"""GPU parity of the result routes on ONE device: every entry point that stores results for other GPUs (kc_vote_i32_peers,
kc_vote_i32_peers_packed, kc_vote_i32_wire, kc_numeric_f64_peers, kc_push_results), and the kernels only those routes launch,
against the C oracle bit for bit.

A route stores each result at `address` and at `address + delta[k]` for every peer k.  Here the peers are MIRROR regions of
one device buffer: the local region and k mirrors, each between guard bands of a sentinel byte, placed so that the deltas
have both signs (ptrs[p] - ptrs[rank] is negative for the ranks below this one).  Every call is then checked three ways:
the local results equal the oracle's; every mirror equals the local region (its mirrored parts; the rest must stay
untouched); every guard band still holds the sentinel.

test_every_dispatched_kernel_runs lists every K1 / K2 / K3b kernel instantiation the dispatch in kllms_b200.cu can reach
(COVERAGE) and checks under torch.profiler that a slice of the inputs here and in test_gpu_kernels.py launches each of them.

Not covered: the multicast route (KC_OUT_MULTIMEM) needs an NVSwitch multicast object; tests/test_gpu_multi.py runs it
on two or more GPUs."""
import ctypes
import re

import numpy as np
import pytest

from oracle import columnar as OC
from tests.helpers import EDGE_EPS, VAL_STYLES, numeric_edge_vals, random_codes, random_vals

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GUARD = 512           # bytes of sentinel before, between and after the regions
VOTE_N = [1, 2, 3, 4, 5, 8, 12, 16, 17, 31, 32, 33, 64]
NUM_N = [1, 2, 3, 4, 5, 8, 11, 16, 24, 32, 48, 64]
F = 6                 # vote fields per record (none_code entries)
RAGGED = [1, 7, 31, 33, 4099 * F]
# over three waves of each TMA kernel's persistent grid on an H100 (132 SMs), so that every warp's pipeline wraps its stages
MANY = {16: 400_003, 32: 400_003, 64: 160_001}


def _torch():
    import torch
    return torch


# ---------------------------------------------------------------- the C ABI through ctypes, and the mirrored buffer

class Abi:
    """The library's C ABI on the current CUDA stream; every call's return code is checked (or returned, with raw=True)."""

    def __init__(self):
        from k_llms_b200 import _native as K
        self.K, self.lib = K, K.load()
        self.stream = _torch().cuda.current_stream().cuda_stream

    def __call__(self, name, *args, raw=False):
        rc = getattr(self.lib, name)(*args, self.stream)
        if raw:
            return rc
        self.K.check(rc)


def deltas_array(deltas):
    return (ctypes.c_int64 * max(len(deltas), 1))(*deltas)


class Mirrored:
    """One device uint8 buffer: the local region and k mirrors of `size` bytes, each between guard bands.  A region is a
    list of segments (name, nbytes, mirrored), each 16-byte aligned; a mirror must equal the local region on the mirrored
    segments and hold the sentinel everywhere else."""

    def __init__(self, segments, k):
        torch = _torch()
        self.seg, off = {}, 0
        for name, nbytes, mirrored in segments:
            self.seg[name] = (off, nbytes, mirrored)
            off += (nbytes + 15) // 16 * 16
        self.size = max(off, 16)
        self.stride = self.size + GUARD
        self.k = k
        self.local = (k + 1) // 2  # mirrors on both sides: deltas of both signs
        self.buf = torch.full((GUARD + (k + 1) * self.stride,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.deltas = [(self.base(r) - self.base(self.local)) for r in range(k + 1) if r != self.local]
        assert all(d % 16 == 0 for d in self.deltas) and (k < 2 or min(self.deltas) < 0 < max(self.deltas))
        self.c_deltas = deltas_array(self.deltas)

    def base(self, r):
        return GUARD + r * self.stride

    def ptr(self, name):
        return self.buf.data_ptr() + self.base(self.local) + self.seg[name][0]

    def view(self, name, dtype):
        off, nbytes, _ = self.seg[name]
        b = self.base(self.local) + off
        return self.buf[b:b + nbytes].view(dtype)

    def fill(self, name, array):
        """Write host bytes into a local segment."""
        torch = _torch()
        off, nbytes, _ = self.seg[name]
        a = np.ascontiguousarray(array).view(np.uint8).reshape(-1)
        assert a.size == nbytes
        b = self.base(self.local) + off
        self.buf[b:b + nbytes].copy_(torch.from_numpy(a))

    def host(self, name, dtype):
        return self.view(name, _torch().uint8).cpu().numpy().view(dtype)

    def check(self):
        """Mirrors and guard bands: the whole buffer must equal the sentinel, with the local segments as they are and the
        mirrored ones copied into every mirror."""
        got = self.buf.cpu().numpy()
        exp = np.full_like(got, SENTINEL)
        lb = self.base(self.local)
        for off, nbytes, mirrored in self.seg.values():
            exp[lb + off:lb + off + nbytes] = got[lb + off:lb + off + nbytes]
            if mirrored:
                for r in range(self.k + 1):
                    exp[self.base(r) + off:self.base(r) + off + nbytes] = got[lb + off:lb + off + nbytes]
        bad = np.nonzero(got != exp)[0]
        if bad.size:
            i = int(bad[0])
            r, o = divmod(i - GUARD, self.stride)
            where = "guard band" if i < GUARD or o >= self.size else next(
                (n for n, (so, nb, _) in self.seg.items() if so <= o < so + nb), "padding")
            raise AssertionError(f"{bad.size} bytes differ; first at region {r} (local = {self.local}) offset {o}: {where}")


def same_numeric(got_val, got_meta, exp_val, exp_meta, what):
    bad = np.nonzero(got_meta != exp_meta)[0]
    assert bad.size == 0, (what, bad.size, bad[:5], OC.meta_fields(got_meta[bad[:1]]), OC.meta_fields(exp_meta[bad[:1]]))
    # NaN outputs ("no value") only need to be NaN on both sides
    ok = (got_val.view(np.uint64) == exp_val.view(np.uint64)) | (np.isnan(got_val) & np.isnan(exp_val))
    assert ok.all(), (what, np.nonzero(~ok)[0][:5])


def wire_overflow(win, meta, wide):
    """Whether some K1 result does not fit the wire (or packed) vote words."""
    w, m = win.astype(np.uint32), meta.astype(np.uint32)
    support, present = (m >> 6) & 0x7F, (m >> 20) & 0x7F
    if wide:
        return bool(((support != 0) & (w >= 1 << 18)).any())
    return bool(((support > 31) | (present > 31) | ((support != 0) & (w > 63))).any())


def num_overflow(meta, wide):
    m = meta.astype(np.uint32)
    return not wide and bool(((((m >> 6) & 0x7F) > 31) | (((m >> 13) & 0x7F) > 31) | (((m >> 20) & 0x7F) > 31)).any())


# ---------------------------------------------------------------- K1 routes

VOTE_ROUTES = ["peers0", "peers1", "peers3", "peers7", "packed3", "wire-narrow0", "wire-narrow3", "wire-wide0", "wire-wide3"]


def run_vote_route(abi, route, codes, none_code, flag):
    """K1 through one non-local route into a fresh mirrored buffer; checks mirrors / guards and returns (win, meta, words)
    with words the packed or wire words (None for the peers route)."""
    torch = _torch()
    G, n = codes.shape
    k = int(route[-1])
    d_codes = torch.from_numpy(codes).cuda()
    d_nc = torch.from_numpy(none_code).cuda() if none_code is not None else None
    nc_ptr, nf = (d_nc.data_ptr(), none_code.size) if none_code is not None else (None, 0)
    flag.zero_()
    if route.startswith("peers"):
        buf = Mirrored([("win", G * 4, True), ("meta", G * 4, True)], k)
        abi("kc_vote_i32_peers", d_codes.data_ptr(), G, n, nc_ptr, nf, buf.ptr("win"), buf.ptr("meta"), k, buf.c_deltas)
        words = None
    elif route.startswith("packed"):
        buf = Mirrored([("win", G * 4, False), ("meta", G * 4, False), ("words", G * 4, True)], k)
        abi("kc_vote_i32_peers_packed", d_codes.data_ptr(), G, n, nc_ptr, nf, buf.ptr("win"), buf.ptr("meta"), buf.ptr("words"),
            k, buf.c_deltas, flag.data_ptr())
        words = np.uint32
    else:
        wide = "wide" in route
        words = np.uint32 if wide else np.uint16
        buf = Mirrored([("win", G * 4, False), ("meta", G * 4, False), ("words", G * (4 if wide else 2), True)], k)
        abi("kc_vote_i32_wire", d_codes.data_ptr(), G, n, nc_ptr, nf, buf.ptr("win"), buf.ptr("meta"), buf.ptr("words"),
            1 if wide else 0, k, buf.c_deltas if k else None, flag.data_ptr())
    buf.check()
    return buf.host("win", np.int32), buf.host("meta", np.uint32), buf.host("words", words) if words else None


def check_vote_route(abi, route, codes, none_code, flag, what):
    from k_llms_b200.distributed import wire_pack_votes
    win, meta, words = run_vote_route(abi, route, codes, none_code, flag)
    exp_win, exp_meta = OC.vote(codes, none_code)
    bad = np.nonzero((win != exp_win) | (meta != exp_meta))[0]
    assert bad.size == 0, (what, bad.size, bad[:5])
    if words is not None:
        wide = words.dtype == np.uint32
        assert np.array_equal(words, wire_pack_votes(exp_win, exp_meta, wide)), what
        assert int(flag.item()) == int(wire_overflow(exp_win, exp_meta, wide)), (what, int(flag.item()))


@pytest.mark.parametrize("route", VOTE_ROUTES)
@pytest.mark.parametrize("n", VOTE_N)
def test_vote_routes_match_oracle(n, route):
    torch = _torch()
    abi = Abi()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(50 * n + VOTE_ROUTES.index(route))
    for G in RAGGED:
        for vocab, p_agree in ((3, 0.6), (1000, 0.3), (60, 0.9)):
            codes = random_codes(rng, G, n, vocab, p_agree=p_agree)
            none_code = np.array([-1, 0, -1, 1, vocab + 5, -1], dtype=np.int32)
            for nc in (None, none_code):
                check_vote_route(abi, route, codes, nc, flag, (G, vocab, nc is not None))


@pytest.mark.parametrize("route", ["peers3", "packed3", "wire-narrow3", "wire-wide3"])
@pytest.mark.parametrize("n", [32, 64])
def test_vote_routes_many_waves(n, route):
    """The TMA vote kernels over several waves of their persistent grid."""
    torch = _torch()
    rng = np.random.default_rng(n)
    codes = random_codes(rng, MANY[n], n, 5)
    none_code = rng.integers(-1, 6, 24).astype(np.int32)
    check_vote_route(Abi(), route, codes, none_code, torch.zeros(1, dtype=torch.int32, device="cuda"), MANY[n])


def boundary_codes():
    """(name, codes [G, n], narrow overflow, wide overflow): results right at the edges of the wire words' fields."""
    full = lambda n, c: np.full((1, n), c, dtype=np.int32)  # noqa: E731
    one_absent = lambda n, c: np.concatenate([full(n - 1, c), full(1, -2)], axis=1)  # noqa: E731
    return [
        ("present 31", one_absent(32, 3), False, False),
        ("present 32", np.concatenate([full(31, 3), full(1, -1)], axis=1), True, False),
        ("support 31", full(31, 5), False, False),
        ("support 32", full(32, 5), True, False),
        ("code 63", full(4, 63), False, False),
        ("code 64", full(4, 64), True, False),
        ("no value, code -1", full(4, -1), False, False),
        ("no value among large codes", np.array([[-1, -2, -1, -1]], dtype=np.int32), False, False),
        ("code 2^18 - 1", full(4, (1 << 18) - 1), True, False),
        ("code 2^18", full(4, 1 << 18), True, True),
        ("code 2^18 beside small results", np.concatenate([full(4, 3)] * 7 + [full(4, 1 << 18)]), True, True),
    ]


@pytest.mark.parametrize("case", [c[0] for c in boundary_codes()])
def test_wire_overflow_flag_boundaries(case):
    """The overflow flag of the narrow and wide wire words and of the packed words is set exactly when a result does not fit
    (support or present > 31 or a code > 63; a code >= 2^18), never by a result without a value."""
    torch = _torch()
    from k_llms_b200.distributed import wire_pack_votes
    abi = Abi()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    _, codes, narrow_over, wide_over = next(c for c in boundary_codes() if c[0] == case)
    exp_win, exp_meta = OC.vote(codes, None)
    assert wire_overflow(exp_win, exp_meta, False) == narrow_over and wire_overflow(exp_win, exp_meta, True) == wide_over
    for route in ("wire-narrow0", "wire-narrow1", "wire-wide0", "wire-wide1", "packed1"):
        win, meta, words = run_vote_route(abi, route, codes, None, flag)
        wide = words.dtype == np.uint32
        assert np.array_equal(win, exp_win) and np.array_equal(meta, exp_meta), route
        assert np.array_equal(words, wire_pack_votes(exp_win, exp_meta, wide)), route
        assert int(flag.item()) == int(wide_over if wide else narrow_over), (route, int(flag.item()))
    # the push kernel packs the same results with the same rule
    G = codes.shape[0]
    pad = (-G) % 8
    win8 = np.concatenate([exp_win, np.full(pad, -1, np.int32)])
    meta8 = np.concatenate([exp_meta, np.zeros(pad, np.uint32)])
    for wide in (False, True):
        flag.zero_()
        slot = run_push(abi, "pack", False, wide, 0, 0, win8, meta8, np.zeros(0), np.zeros(0, np.uint32), flag)
        assert np.array_equal(slot[0], wire_pack_votes(win8, meta8, wide)), wide
        assert int(flag.item()) == int(wide_over if wide else narrow_over), ("push", wide, int(flag.item()))


# ---------------------------------------------------------------- K2 routes

def run_numeric_peers(abi, vals, rel, ab, k):
    torch = _torch()
    G, n = vals.shape
    d_vals = torch.from_numpy(vals).cuda()
    buf = Mirrored([("value", G * 8, True), ("meta", G * 4, True)], k)
    abi("kc_numeric_f64_peers", d_vals.data_ptr(), G, n, float(rel), float(ab), buf.ptr("value"), buf.ptr("meta"), k, buf.c_deltas)
    buf.check()
    return buf.host("value", np.float64), buf.host("meta", np.uint32)


@pytest.mark.parametrize("k", [0, 1, 3, 7])
@pytest.mark.parametrize("n", NUM_N)
def test_numeric_peers_match_oracle(n, k):
    abi = Abi()
    rng = np.random.default_rng(30 * n + k)
    for style in VAL_STYLES:
        vals = random_vals(rng, 4099 * 2, n, style)  # 2 numeric fields per record
        for rel, ab in EDGE_EPS:
            with np.errstate(all="ignore"):
                exp_val, exp_meta = OC.numeric(vals, rel, ab)
            same_numeric(*run_numeric_peers(abi, vals, rel, ab, k), exp_val, exp_meta, (style, rel, ab))
    for G in RAGGED:
        vals = random_vals(rng, G, n, "near")
        same_numeric(*run_numeric_peers(abi, vals, 0.03, 1e-6, k), *OC.numeric(vals), G)


@pytest.mark.parametrize("n", [16, 32])
def test_numeric_peers_edges(n):
    """test_gpu_kernels.py::test_numeric_fast_path_edges's inputs through the general TMA kernels (the peers route does not
    take the fast kernels): their tie and low-bit repair paths at the edges."""
    abi = Abi()
    vals = numeric_edge_vals(np.random.default_rng(900 + n), 20000, n)
    for k in (1, 3):
        for rel, ab in EDGE_EPS:
            with np.errstate(all="ignore"):
                exp_val, exp_meta = OC.numeric(vals, rel, ab)
            same_numeric(*run_numeric_peers(abi, vals, rel, ab, k), exp_val, exp_meta, (k, rel, ab))


@pytest.mark.parametrize("n", [16, 32, 64])
def test_numeric_peers_many_waves(n):
    """The general TMA K2 kernels over several waves of their persistent grid."""
    rng = np.random.default_rng(n)
    vals = random_vals(rng, MANY[n], n, "lowbits")
    same_numeric(*run_numeric_peers(Abi(), vals, 0.03, 1e-6, 3), *OC.numeric(vals), MANY[n])


# ---------------------------------------------------------------- kc_push_results

def run_push(abi, mode, alias, wide, k, max_ctas, win, vmeta, value, nmeta, flag, codes=None):
    """kc_push_results into a mirrored slot.  mode "pack": the K1 results (win, vmeta) are given; mode "wire": K1 wrote the
    wire words into the slot first (kc_vote_i32_wire on `codes`; win / vmeta are what it must compute).  alias: the values
    already sit in the slot (K2 wrote them there) instead of a separate array.  Returns the slot's (vote words, values,
    numeric words) after checking mirrors and guard bands."""
    torch = _torch()
    gv, gx = win.size, value.size
    wb = 4 if wide else 2
    buf = Mirrored([("votes", gv * wb, True), ("value", gx * 8, True), ("nwords", gx * wb, True)], k)
    d_win = torch.from_numpy(win).cuda()
    d_vmeta = torch.from_numpy(vmeta.view(np.int32)).cuda()
    d_nmeta = torch.from_numpy(nmeta.view(np.int32)).cuda()
    d_value = torch.from_numpy(value).cuda()
    if alias:
        buf.fill("value", value)
        value_ptr = buf.ptr("value")
    else:
        value_ptr = d_value.data_ptr()
    if mode == "wire":
        n = codes.shape[1]
        kwin, kmeta = torch.empty_like(d_win), torch.empty_like(d_vmeta)
        d_codes = torch.from_numpy(codes).cuda()
        abi("kc_vote_i32_wire", d_codes.data_ptr(), gv, n, None, 0, kwin.data_ptr(), kmeta.data_ptr(), buf.ptr("votes"),
            1 if wide else 0, 0, None, flag.data_ptr())
        assert np.array_equal(kwin.cpu().numpy(), win) and np.array_equal(kmeta.cpu().numpy().view(np.uint32), vmeta)
        win_ptr = meta_ptr = None
    else:
        win_ptr, meta_ptr = d_win.data_ptr(), d_vmeta.data_ptr()
    abi("kc_push_results", win_ptr, meta_ptr, gv, value_ptr, d_nmeta.data_ptr(), gx, buf.ptr("votes"), buf.ptr("value"),
        buf.ptr("nwords"), 1 if wide else 0, k, buf.c_deltas, flag.data_ptr(), max_ctas)
    buf.check()
    wt = np.uint32 if wide else np.uint16
    return buf.host("votes", wt), buf.host("value", np.float64), buf.host("nwords", wt)


@pytest.mark.parametrize("max_ctas", [1, 0], ids=["one-cta", "grid"])
@pytest.mark.parametrize("k", [0, 3])
@pytest.mark.parametrize("wide", [False, True], ids=["narrow", "wide"])
@pytest.mark.parametrize("alias", [True, False], ids=["value-in-slot", "value-apart"])
@pytest.mark.parametrize("mode", ["pack", "wire"])
def test_push_results(mode, alias, wide, k, max_ctas):
    """The slot and every mirror equal the packing of the oracle's results, and decode to the library's confidences of the
    full result words."""
    torch = _torch()
    from k_llms_b200 import _native as K
    from k_llms_b200.distributed import wire_confidences, wire_pack_num, wire_pack_votes
    abi = Abi()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(7)
    n = 40 if wide else 16
    gv, gx = 8 * 4099, 8 * 1031
    codes = random_codes(rng, gv, n, 2000 if wide else 40, p_agree=0.7)
    vals = random_vals(rng, gx, n, "near")
    win, vmeta = OC.vote(codes, None)
    value, nmeta = OC.numeric(vals)
    words, got_value, nwords = run_push(abi, mode, alias, wide, k, max_ctas, win, vmeta, value, nmeta, flag, codes=codes)
    assert np.array_equal(words, wire_pack_votes(win, vmeta, wide))
    assert np.array_equal(got_value.view(np.uint64), value.view(np.uint64))
    assert np.array_equal(nwords, wire_pack_num(nmeta, wide))
    assert int(flag.item()) == int(wire_overflow(win, vmeta, wide) or num_overflow(nmeta, wide))
    vconf, nconf = wire_confidences(words, nwords, wide)
    to_dev = lambda m: torch.from_numpy(m.view(np.int32)).cuda()  # noqa: E731
    assert np.array_equal(vconf, K.confidence(to_dev(vmeta), False).cpu().numpy())
    assert np.array_equal(nconf, K.confidence(to_dev(nmeta), True).cpu().numpy())


def test_push_results_one_segment():
    """Only vote results, then only numeric results: the empty segments are skipped."""
    torch = _torch()
    from k_llms_b200.distributed import wire_pack_num, wire_pack_votes
    abi = Abi()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(8)
    win, vmeta = OC.vote(random_codes(rng, 8 * 33, 16, 7), None)
    value, nmeta = OC.numeric(random_vals(rng, 8 * 33, 16, "ints"))
    none_i, none_u, none_f = np.zeros(0, np.int32), np.zeros(0, np.uint32), np.zeros(0)
    words, _, nwords = run_push(abi, "pack", False, False, 3, 0, win, vmeta, none_f, none_u, flag)
    assert np.array_equal(words, wire_pack_votes(win, vmeta, False)) and nwords.size == 0
    words, got_value, nwords = run_push(abi, "pack", True, False, 3, 0, none_i, none_u, value, nmeta, flag)
    assert words.size == 0 and np.array_equal(nwords, wire_pack_num(nmeta, False))
    assert np.array_equal(got_value.view(np.uint64), value.view(np.uint64))


# ---------------------------------------------------------------- argument checks (nothing is launched)

def test_route_argument_checks():
    torch = _torch()
    from k_llms_b200 import _native as K
    abi = Abi()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda").data_ptr()
    eight = deltas_array([4096] * 8)
    odd8, odd16 = deltas_array([4096, 4100]), deltas_array([4096, 4104])
    EINVAL = K.KC_EINVAL
    # n_peers = 8: more peers than a route has delta slots
    assert abi("kc_vote_i32_peers", p, 64, 4, None, 0, p, p, 8, eight, raw=True) == EINVAL
    assert abi("kc_vote_i32_peers_packed", p, 64, 4, None, 0, p, p, p, 8, eight, flag, raw=True) == EINVAL
    assert abi("kc_vote_i32_wire", p, 64, 4, None, 0, p, p, p, 0, 8, eight, flag, raw=True) == EINVAL
    assert abi("kc_numeric_f64_peers", p, 64, 4, 0.03, 1e-6, p, p, 8, eight, raw=True) == EINVAL
    assert abi("kc_push_results", p, p, 64, p, p, 64, p, p, p, 0, 8, eight, flag, 0, raw=True) == EINVAL
    # deltas: multiples of 8 bytes for the kernels' scalar stores, of 16 for the push kernel's vectors
    assert abi("kc_vote_i32_peers", p, 64, 4, None, 0, p, p, 2, odd8, raw=True) == EINVAL
    assert abi("kc_numeric_f64_peers", p, 64, 4, 0.03, 1e-6, p, p, 2, odd8, raw=True) == EINVAL
    assert abi("kc_push_results", p, p, 64, p, p, 64, p, p, p, 0, 2, odd16, flag, 0, raw=True) == EINVAL
    # push: whole 16-byte vectors of results
    assert abi("kc_push_results", p, p, 60, p, p, 64, p, p, p, 0, 0, None, flag, 0, raw=True) == EINVAL
    assert abi("kc_push_results", p, p, 64, p, p, 12, p, p, p, 0, 0, None, flag, 0, raw=True) == EINVAL
    # the TMA kernels' field map stops below 60000 fields
    codes = torch.zeros((60000, 32), dtype=torch.int32, device="cuda")
    nc = torch.zeros(60000, dtype=torch.int32, device="cuda")
    out = torch.zeros(2 * 60000, dtype=torch.int32, device="cuda")
    c, w, m = codes.data_ptr(), out.data_ptr(), out.data_ptr() + 60000 * 4
    assert abi("kc_vote_i32", c, 60000, 32, nc.data_ptr(), 60000, w, m, raw=True) == EINVAL
    assert abi("kc_vote_i32_peers", c, 60000, 32, nc.data_ptr(), 60000, w, m, 0, None, raw=True) == EINVAL
    torch.cuda.synchronize()
    assert not buf.any() and not out.any(), "a rejected call stored something"


# ---------------------------------------------------------------- every dispatched kernel runs

def _both(fmt):
    return [fmt.format(nc=nc) for nc in ("false", "true")]


# Every kernel instantiation kc_vote_i32* / kc_vote_i8 / kc_numeric_f64* / kc_weighted_vote_i32 / kc_push_results can launch,
# local and non-local routes, read off their dispatch in kllms_b200.cu (template arguments as the demangled names print them).
COVERAGE = (
    # K1, local n = 2, 4, 8: GPT groups per thread, the last < GPT groups one per thread (also the non-local n = 2, 4, 8)
    _both("vote_multi_kernel<2,8,{nc}>") + _both("vote_multi_kernel<4,4,{nc}>") + _both("vote_multi_kernel<8,2,{nc}>")
    + _both("vote_direct_kernel<int,2,true,{nc},false>") + _both("vote_direct_kernel<int,4,true,{nc},true>")
    + _both("vote_direct_kernel<int,8,true,{nc},true>")
    # K1 n = 1, 16; n = 32, 64 (TMA); other n: the next power of two, cells beyond n absent
    + _both("vote_direct_kernel<int,1,true,{nc},false>") + _both("vote_direct_kernel<int,16,true,{nc},true>")
    + _both("vote_tma_kernel<32,8,2,{nc}>") + _both("vote_tma_kernel<64,4,2,{nc}>")
    + [s for np_ in (4, 8, 16, 32, 64) for s in _both(f"vote_direct_kernel<int,{np_},false,{{nc}},false>")]
    # K1 on int8 cells (never PREFETCH)
    + [s for np_ in (4, 8, 16, 32, 64) for vec in ("false", "true")
       for s in _both(f"vote_direct_kernel<signedchar,{np_},{vec},{{nc}},false>")]
    # K2 local: n = 2, 4 (+ their one-group tails), 8, 16, 32 fast kernels
    + ["numeric_pairs_kernel", "numeric_quads_kernel", "numeric_direct_fast_kernel<8,128>", "numeric_tma_fast_kernel<16,4,1,6>",
       "numeric_tma_fast_kernel<32,4,1,4>"]
    # K2 general kernels: n = 16, 32 non-local, n = 64 both; direct kernels for the other n (PREFETCH where n == NP in {4, 8})
    + ["numeric_tma_kernel<16,4,1,7>", "numeric_tma_kernel<32,4,1,4>", "numeric_tma_kernel<64,2,1,3>",
       "numeric_direct_kernel<2,128,false>", "numeric_direct_kernel<4,128,false>", "numeric_direct_kernel<4,128,true>",
       "numeric_direct_kernel<8,128,false>", "numeric_direct_kernel<8,128,true>", "numeric_direct_kernel<16,128,false>",
       "numeric_direct_kernel<32,128,false>", "numeric_direct_kernel<64,64,false>"]
    # K3b: n < 8; the per-record kernel; n = 32 / 64 below 60000 fields (n = 32 with a weight pre-pass from 5 fields on)
    + ["weighted_vote_kernel<2>", "weighted_vote_kernel<4>", "weighted_vote_kernel<8>", "weighted_vote_rec_kernel<8,128>",
       "weighted_vote_rec_kernel<16,128>", "weighted_vote_rec_kernel<32,128>", "weighted_vote_rec_kernel<64,128>",
       "weight_rows_kernel<32>", "weighted_vote_rows_kernel<32,8,2,3>", "weighted_vote_tma_kernel<32,8,2,3,true>",
       "weighted_vote_tma_kernel<64,4,2,3,false>"]
    + ["push_kernel"]
)


def _kernel_key(name):
    """'void kc::vote_tma_kernel<32, 8, 2, true>(CUtensorMap_st, ...)' -> 'vote_tma_kernel<32,8,2,true>'."""
    m = re.search(r"kc::(\w+(?:<[^()]*>)?)\(", name)
    return m.group(1).replace(" ", "") if m else None


def test_every_dispatched_kernel_runs():
    torch = _torch()
    from torch.profiler import ProfilerActivity, profile
    from k_llms_b200 import _native as K
    abi = Abi()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(1)
    G = 4099 * F + 1  # odd: every multi-group kernel leaves a tail
    none_code = np.array([-1, 0, -1, 1, 7, -1], dtype=np.int32)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for n in VOTE_N:
            codes = random_codes(rng, G, n, 5)
            for nc in (None, none_code):
                check_vote_route(abi, "peers1", codes, nc, flag, n)
                ew, em = OC.vote(codes, nc)
                w, m = vote_local(abi, codes, nc)
                assert np.array_equal(w.cpu().numpy(), ew) and np.array_equal(m.cpu().numpy().view(np.uint32), em), n
                w8, m8 = K.vote_i8(torch.from_numpy(codes.astype(np.int8)).cuda(), torch.from_numpy(nc).cuda() if nc is not None else None)
                assert np.array_equal(w8.cpu().numpy(), ew) and np.array_equal(m8.cpu().numpy().view(np.uint32), em), n
        for n in NUM_N:
            vals = random_vals(rng, 4099, n, "near")
            ev, em = OC.numeric(vals)
            same_numeric(*run_numeric_peers(abi, vals, 0.03, 1e-6, 1), ev, em, n)
            v, m = K.numeric(torch.from_numpy(vals).cuda())
            same_numeric(v.cpu().numpy(), m.cpu().numpy().view(np.uint32), ev, em, n)
        for n, fields in ((2, 5), (4, 5), (6, 5), (8, 5), (12, 5), (24, 5), (48, 5), (32, 24), (32, 4), (64, 24)):
            codes = random_codes(rng, 301 * fields, n, 4).reshape(301, fields, n)
            lp = (-rng.exponential(4.0, (301, n))).astype(np.float32)
            ew, em, ewt = OC.weighted_vote(codes, lp)
            w, m, wt = K.weighted_vote(torch.from_numpy(codes).cuda(), torch.from_numpy(lp).cuda())
            assert np.array_equal(w.cpu().numpy(), ew) and np.array_equal(wt.cpu().numpy().view(np.uint32), ewt.view(np.uint32))
        win, vmeta = OC.vote(random_codes(rng, 64, 16, 5), None)
        value, nmeta = OC.numeric(random_vals(rng, 64, 16, "ints"))
        run_push(abi, "pack", False, False, 1, 0, win, vmeta, value, nmeta, flag)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if not names:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable)")
    seen = {k for k in map(_kernel_key, names) if k}
    missing = [k for k in COVERAGE if k not in seen]
    assert not missing, (missing, sorted(seen))
    assert len(set(COVERAGE)) == len(COVERAGE)


def vote_local(abi, codes, none_code):
    """K1 through the plain entry point, also on group counts that end inside a record (the Python wrapper wants whole
    records)."""
    torch = _torch()
    G, n = codes.shape
    d_codes = torch.from_numpy(codes).cuda()
    d_nc = torch.from_numpy(none_code).cuda() if none_code is not None else None
    win = torch.empty(G, dtype=torch.int32, device="cuda")
    meta = torch.empty(G, dtype=torch.int32, device="cuda")
    abi("kc_vote_i32", d_codes.data_ptr(), G, n, d_nc.data_ptr() if d_nc is not None else None, 0 if d_nc is None else none_code.size,
        win.data_ptr(), meta.data_ptr())
    return win, meta
