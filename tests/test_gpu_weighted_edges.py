"""GPU: every K3b kernel (DESIGN.md §5) on the weighted vote's decision edges, against the brute force of
tests/test_weighted_edges_host.py (every class summed in index order, no walk, no early stop) and the C oracle.

The families (exact fp32 ties in every visiting order, order-sensitive near-ties, the stopping bound within ulps, the
record's heaviest candidate None / absent / losing / tied, clamped weights, rows with one cell knocked out at lanes 0, 31, 32,
63) go through kc_weighted_vote_i32 with and without a none_code table at every n that picks another kernel, and through
kc_weighted_vote_groups_i8 with shuffled group_record.  Each test checks under torch.profiler that the kernels it means to
test ran, and counts on the host how many groups wv_first_pass leaves to the warp walk, so that a generator change cannot
quietly make the cases easy."""
import json

import numpy as np
import pytest

from oracle import columnar as OC
from tests import test_weighted_edges_host as H
from tests.helpers import assert_kernels_ran, kernels_seen, profiled

pytestmark = pytest.mark.gpu

N_LIST = [1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17, 31, 32, 33, 63, 64]
F_LIST = [1, 2, 3, 4, 5, 6, 7, 31, 32, 33]  # records on both sides of the n = 32 rows / TMA switch, partial last tiles
GROUPS = 6000  # per family, none_code mode and field count
WALK_FLOOR = 1000  # groups per TMA kernel that wv_first_pass must leave to wv_warp_walk


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _pow2(n, lo):
    p = lo
    while p < n:
        p *= 2
    return p


def i32_kernels(n, F):
    """The kernels kc_weighted_vote_i32 launches for n candidates and F fields per record."""
    if n in (32, 64) and F < 60000:
        if n == 32 and min(32, 31 // F + 2) <= 8:
            return ["weight_rows_kernel<32>", "weighted_vote_rows_kernel<32,8,2,3>"]
        return ["weighted_vote_tma_kernel<32,8,2,3,true>" if n == 32 else "weighted_vote_tma_kernel<64,4,2,3,false>"]
    if n < 8:
        return [f"weighted_vote_kernel<{2 if n <= 2 else 4 if n <= 4 else 8}>"]
    return [f"weighted_vote_rec_kernel<{_pow2(n, 8)},128>"]


def groups_kernels(n):
    np_ = _pow2(n, 4)
    return [f"weight_rows_n_kernel<{np_}>", f"weighted_vote_groups_kernel<{np_},{'true' if n == np_ else 'false'}>"]


def run_i32(codes, seq, nc):
    torch = _torch()
    from k_llms_b200 import _native as K
    w, m, wt = K.weighted_vote(torch.from_numpy(codes).cuda(), torch.from_numpy(seq).cuda(),
                               torch.from_numpy(nc).cuda() if nc is not None else None)
    torch.cuda.synchronize()
    return dict(win=w.cpu().numpy(), meta=m.cpu().numpy().view(np.uint32), weight=wt.cpu().numpy())


def run_groups(codes8, rec, seq):
    torch = _torch()
    from k_llms_b200 import _native as K
    w, m, wt = K.weighted_vote_groups(torch.from_numpy(codes8).cuda(), torch.from_numpy(rec).cuda(), torch.from_numpy(seq).cuda())
    torch.cuda.synchronize()
    return dict(win=w.cpu().numpy(), meta=m.cpu().numpy().view(np.uint32), weight=wt.cpu().numpy())


def check_case(codes, seq, nc, what, ref=None):
    """kc_weighted_vote_i32 against the brute force (every output, tie flag, weight bits) and the C oracle; returns the
    brute force's results and the per-group rows."""
    c2, s2, nc2 = H.flat(codes, seq, nc)
    ref = H.brute(c2, s2, nc2) if ref is None else ref
    got = run_i32(codes, seq, nc)
    H.check_against(got, ref, ("kc_weighted_vote_i32",) + what)
    ew, em, ewt = OC.weighted_vote(codes, seq, nc)
    H.check_against(dict(win=ew, meta=em, weight=ewt), ref, ("C oracle",) + what)
    return ref, (c2, s2, nc2)


def check_groups(rng, codes, seq, ref, what):
    """The same cells through kc_weighted_vote_groups_i8 (int8, no none_code) with the groups in shuffled order."""
    R, F, n = codes.shape
    perm = rng.permutation(R * F)
    rec = (np.arange(R * F, dtype=np.int32) // F)[perm]
    got = run_groups(np.ascontiguousarray(codes.reshape(R * F, n)[perm].astype(np.int8)), rec, seq)
    H.check_against(got, {k: ref[k][perm] for k in ("win", "meta", "weight")}, ("kc_weighted_vote_groups_i8",) + what)


def _fields(n, family, with_nc):
    f = F_LIST[(2 * family + int(with_nc) + n) % len(F_LIST)]
    if n != 32:
        return [f]
    # n = 32: every family on both sides of the switch (TMA below 5 fields, the weight-row pre-pass from 5 on)
    return [f, F_LIST[(2 * family + int(with_nc)) % 4], F_LIST[4 + (2 * family + int(with_nc)) % 6]]


@pytest.mark.parametrize("n", N_LIST)
def test_every_k3b_kernel_on_the_edge_families(n):
    _torch()
    rng = np.random.default_rng(31000 + n)
    expected = set(groups_kernels(n))
    undecided, ties = {}, 0
    with profiled() as prof:
        for family in (1, 2, 3, 4, 5, 6):
            pool = H.design_pool(rng, family, n)
            for with_nc in (False, True):
                for F in sorted(set(_fields(n, family, with_nc))):
                    R = max(2, GROUPS // F)
                    codes, seq, nc = H.make_case(rng, family, n, R, F, with_nc, pool)
                    what = (family, n, F, with_nc)
                    ref, rows = check_case(codes, seq, nc, what)
                    kernels = i32_kernels(n, F)
                    expected.update(kernels)
                    ties += int(((ref["meta"] >> 29) & 1).sum())
                    if "tma" in kernels[-1] or "rows" in kernels[-1]:
                        undecided[kernels[-1]] = undecided.get(kernels[-1], 0) + int(H.first_pass(*rows, ref).sum())
                    if not with_nc:
                        check_groups(rng, codes, seq, ref, what)
    assert_kernels_ran(prof, expected)
    print(f"\nn={n}: groups with the tie flag {ties}; groups wv_first_pass leaves to the warp walk {undecided}")
    assert ties >= 500 or n == 1, ties  # one cell cannot tie
    for k, v in undecided.items():
        assert v >= WALK_FLOOR, (k, undecided)


def test_rows_kernel_cycles_weight_slots():
    """n = 32 at 6 fields: enough tiles that every warp of weighted_vote_rows_kernel wraps its three weight slots several
    times (about 26,000 tiles over at most 132 x 3 CTAs of 8 warps).  Every group against the C oracle, a sample against the
    brute force."""
    _torch()
    rng = np.random.default_rng(3232)
    n, F = 32, 6
    parts = [H.make_case(rng, fam, n, 35_000, F, fam % 2 == 0) for fam in (1, 2, 3, 4)]
    codes = np.concatenate([p[0] for p in parts])
    seq = np.concatenate([p[1] for p in parts])
    nc = np.where(np.arange(F) % 2 == 0, -1, rng.integers(0, 128, F)).astype(np.int32)
    with profiled() as prof:
        got = run_i32(codes, seq, nc)
    assert_kernels_ran(prof, i32_kernels(n, F))
    ew, em, ewt = OC.weighted_vote(codes, seq, nc)
    H.check_against(got, dict(win=ew, meta=em, weight=ewt), "rows kernel, all groups")
    c2, s2, nc2 = H.flat(codes, seq, nc)
    pick = rng.choice(len(c2), 60_000, replace=False)
    ref = H.brute(c2[pick], s2[pick], nc2[pick])
    H.check_against({k: v[pick] for k, v in got.items()}, ref, "rows kernel, sample")
    walked = int(H.first_pass(c2[pick], s2[pick], nc2[pick], ref).sum())
    assert walked >= WALK_FLOOR, walked


@pytest.mark.parametrize("n", [32, 64])
def test_many_fields_fallback_on_the_edges(n):
    """60000 fields per record send n = 32 and 64 to the per-record kernel: all-near-1 and clamped weights, with a
    none_code table."""
    _torch()
    rng = np.random.default_rng(60000 + n)
    F = 60000
    pool = [H.design_near_one(rng, n), H.design_clamped(rng, n)]
    codes, seq, nc = H.make_case(rng, 3, n, 2, F, True, pool=[(None, p[1], p[2]) for p in pool])
    with profiled() as prof:
        ref, _ = check_case(codes, seq, nc, ("fallback", n))
    assert_kernels_ran(prof, i32_kernels(n, F))
    assert i32_kernels(n, F) == [f"weighted_vote_rec_kernel<{n},128>"]
    assert int(((ref["meta"] >> 29) & 1).sum()) >= 100


@pytest.mark.parametrize("F", [4, 5])
def test_rows_kernel_switch_at_five_fields(F):
    """n = 32 switches from the TMA kernel to the weight-row pre-pass once a tile of 32 groups spans at most 8 records:
    rec_cap = min(32, 31 / F + 2) <= 8 from F = 5 on."""
    _torch()
    rng = np.random.default_rng(F)
    codes, seq, nc = H.make_case(rng, 1, 32, 400, F, False)
    with profiled() as prof:
        check_case(codes, seq, nc, ("switch", F))
    seen, any_names = kernels_seen(prof)
    if not any_names:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable)")
    rows = "weighted_vote_rows_kernel<32,8,2,3>" in seen
    tma = "weighted_vote_tma_kernel<32,8,2,3,true>" in seen
    assert (rows, tma) == ((True, False) if F >= 5 else (False, True)), sorted(seen)


@pytest.mark.parametrize("n", [3, 8, 32])
def test_device_json_path_on_the_edge_families(n):
    """Records built from families 1 (ties), 4 (the heaviest candidate) and 5 (clamped weights) through
    kc_consolidate_json_packed_weighted: value and printed likelihood byte for byte against the weighted oracle."""
    _torch()
    from k_llms_b200 import _native as K
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from k_llms_b200.utils.consolidation import _aligned_sync, _format_consensus_content, _safe_parse_content
    from oracle import consensus_py as O
    from tests import weighted_oracle as W
    embed = lambda texts: [[0.0] for _ in texts]  # noqa: E731
    rng = np.random.default_rng(555 + n)
    F = 3
    parts = [H.make_case(rng, fam, n, 150, F, False) for fam in (1, 4, 5)]
    codes = np.concatenate([p[0] for p in parts])
    seq = np.concatenate([p[1] for p in parts])
    records = []
    for r in range(len(codes)):
        records.append([json.dumps({f"f{f}": (f"v{int(codes[r, f, c])}" if codes[r, f, c] >= 0 else None) for f in range(F)})
                        for c in range(n)])
    blob, off, _ = K.pack_texts(records)
    res = K.consolidate_json_packed_weighted(blob, off, n, seq.reshape(-1))
    try:
        got = res.pairs()
        on_device = 0
        for r, (texts, p) in enumerate(zip(records, got)):
            if p is None:
                continue
            on_device += 1
            contents = [_safe_parse_content(t) for t in texts]
            aligned = _aligned_sync(contents, ConsensusSettings(), embed, None)
            value, conf = W.client_order(contents, seq[r], O.DEFAULTS, embed, aligned=aligned)
            assert p == (_format_consensus_content(value), json.dumps(conf)), (r, texts, seq[r], p, value, conf)
        assert on_device >= 0.9 * len(records), (on_device, len(records))
    finally:
        res.close()
