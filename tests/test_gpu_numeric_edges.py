"""GPU: every K2 kernel (kc_numeric.cuh) on the numeric clustering's decision edges, against the brute force of
tests/test_numeric_edges_host.py (the reference's numeric branch restated over K2's cells, with numpy's own mean, median and
std).

The families (majorities at 2c = m - 1 .. m + 2 with every census mix and single cells at lanes 0, 31, 32, 63; neighbours at
and around the tolerance edge, uncertifiable from their high word or sharing one; the walk's extras in every split and the
cells beyond them; clusters whose numpy mean a left-to-right sum or a misplaced extra would change (also in full at n = 16
and 32: every (z mod 8, nb, na) on the fast path); low-bit repairs, chain
edges across zero, +-1.7e308, majorities ending or starting at the middle element, n = 64 clusters on both sides of mask bit
32; ties decided by support, spread, |center| and order; the n = 2 and n = 4 tables) run through kc_numeric_f64 at every n
that selects another kernel or padding, with group counts that leave the pairs and quads kernels a tail, through
kc_numeric_f64_peers, tiled past three waves of the persistent grids, and as {"x": number} records through the device JSON
path and H1.  Family 8 (per-tile deferral layouts) drives the fast kernels' deferral queues to exactly 32, past it (the
overflow re-read from global memory) and to final drains of 1 and 31.  Every value and result word must equal the brute
force's bit for bit; a NaN with no value only needs to be NaN on both sides."""
import json

import numpy as np
import pytest

from oracle import columnar as OC
from tests import test_numeric_edges_host as H
from tests.helpers import EDGE_EPS, assert_kernels_ran, consolidate_json_with_oracle, jsongpu_with_oracle, profiled, same

pytestmark = pytest.mark.gpu

MANY = {16: 400_003, 32: 400_003, 64: 160_001}  # over three waves of each TMA kernel's persistent grid on an H100 (132 SMs)
QUEUE_MANY = {8: 800_031, 16: 400_031, 32: 400_001}  # several tiles per warp of the fast kernels: the queues overflow


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def kernels(n, G, local=True):
    """The K2 kernels kc_numeric_f64 (local) or kc_numeric_f64_peers launches for G groups of n cells
    (test_gpu_routes.COVERAGE)."""
    NP = H.pow2(n)
    direct = f"numeric_direct_kernel<{NP},{64 if NP == 64 else 128},{'true' if n == NP and n in (4, 8) else 'false'}>"
    if local:
        if n == 2:
            return ["numeric_pairs_kernel"] + (["numeric_direct_kernel<2,128,false>"] if G % 4 else [])
        if n == 4:
            return ["numeric_quads_kernel"] + (["numeric_direct_kernel<4,128,true>"] if G % 2 else [])
        if n == 8:
            return ["numeric_direct_fast_kernel<8,128>"]
        if n in (16, 32):
            return [f"numeric_tma_fast_kernel<{n},4,1,{6 if n == 16 else 4}>"]
    if n in (16, 32, 64):
        return [f"numeric_tma_kernel<{n},{2 if n == 64 else 4},1,{7 if n == 16 else 4 if n == 32 else 3}>"]
    return [direct]


def run_local(vals, rel, ab):
    torch = _torch()
    from k_llms_b200 import _native as K
    v, m = K.numeric(torch.from_numpy(np.ascontiguousarray(vals).view(np.float64)).cuda(), rel, ab)
    return v.cpu().numpy().view(np.uint64), m.cpu().numpy().view(np.uint32)


def run_peers(vals, rel, ab):
    from tests.test_gpu_routes import Abi, run_numeric_peers
    v, m = run_numeric_peers(Abi(), np.ascontiguousarray(vals).view(np.float64), rel, ab, 1)
    return v.view(np.uint64), m


def edge_rows(n, i):
    """The host file's rows at n under EDGE_EPS[i], and their first three again: a group count that is odd and not a
    multiple of 4, so the pairs and quads kernels leave a tail to the direct kernel."""
    vals, _ = H._rows(n, i)
    return np.ascontiguousarray(np.concatenate([vals, vals[:3]]))


def test_edge_kernels_cover_every_k2_instantiation():
    """The kernels the family test expects, over every n and both routes, are all 16 K2 instantiations of COVERAGE."""
    from tests.test_gpu_routes import COVERAGE
    k2 = {k for k in COVERAGE if k.startswith("numeric_")}
    want = {k for n in H.N_LIST for local in (True, False) for k in kernels(n, len(edge_rows(n, 0)), local)}
    assert len(k2) == 16 and want == k2, (sorted(k2 - want), sorted(want - k2))


@pytest.mark.parametrize("n", H.N_LIST)
def test_every_k2_kernel_on_the_edge_families(n):
    _torch()
    expected = set()
    with profiled() as prof:
        for i, (rel, ab) in enumerate(EDGE_EPS):
            vals = edge_rows(n, i)
            ev, em, _ = H.brute(vals, rel, ab)
            H.check_against(*run_local(vals, rel, ab), ev, em, ("kc_numeric_f64", n, rel, ab), vals)
            H.check_against(*run_peers(vals, rel, ab), ev, em, ("kc_numeric_f64_peers", n, rel, ab), vals)
            expected.update(kernels(n, len(vals)) + kernels(n, len(vals), local=False))
    assert_kernels_ran(prof, expected)
    print(f"\nn={n}: {len(vals)} groups x {len(EDGE_EPS)} settings; kernels {sorted(expected)}")


@pytest.mark.parametrize("n", [16, 32])
def test_fast_kernels_on_the_summation_order_rows(n):
    """Family 4 in full: every cluster sum_order_cases finds, one row each, under every EDGE_EPS setting, through the fast
    kernel and the general one (peers route).  On the host, test_summation_order_rows counts that these rows reach every
    (z mod 8, nb, na) on the fast path."""
    _torch()
    with profiled() as prof:
        for i, (rel, ab) in enumerate(EDGE_EPS):
            vals, _ = H.sum_order_rows(n, i)
            ev, em, _ = H.brute(vals, rel, ab)
            H.check_against(*run_local(vals, rel, ab), ev, em, ("sum order, kc_numeric_f64", n, rel, ab), vals)
            H.check_against(*run_peers(vals, rel, ab), ev, em, ("sum order, kc_numeric_f64_peers", n, rel, ab), vals)
    assert_kernels_ran(prof, kernels(n, len(vals)) + kernels(n, len(vals), local=False))


@pytest.mark.parametrize("n", [16, 32, 64])
def test_k2_kernels_over_many_waves(n):
    """The families tiled past three waves of the persistent TMA grids, under the default and the exact tolerance, through
    both routes: every group against the brute force."""
    _torch()
    for i in (0, 1):
        rel, ab = EDGE_EPS[i]
        base = edge_rows(n, i)
        ev, em, _ = H.brute(base, rel, ab)
        pick = np.arange(MANY[n]) % len(base)
        big = np.ascontiguousarray(base[pick])
        with profiled() as prof:
            local = run_local(big, rel, ab)
            peers = run_peers(big, rel, ab)
        assert_kernels_ran(prof, kernels(n, MANY[n]) + kernels(n, MANY[n], local=False))
        H.check_against(*local, ev[pick], em[pick], ("many waves, local", n, rel, ab))
        H.check_against(*peers, ev[pick], em[pick], ("many waves, peers", n, rel, ab))


@pytest.mark.parametrize("n", [8, 16, 32])
def test_fast_kernels_deferral_queues(n):
    """Family 8: per-tile deferral counts of 0, 1, 2, 16, 31 and 32 on their own and mixed, at 32t + 1 and 32t + 31 groups
    (one tile per warp: the final drain holds that tile's deferred groups) and at several tiles per warp (the queue
    passes 32 and re-reads its overflow).  Every group holds a value of its own, so a result stored at another index
    shows."""
    _torch()
    rel, ab = EDGE_EPS[0]
    with profiled() as prof:
        for name, lay in H.QUEUE_LAYOUTS.items():
            for G in (32 * 5 + 1, 32 * 5 + 31, 32 * 40 + 1):
                vals = H.queue_rows(n, G, lay, G + n)
                ev, em, _ = H.brute(vals, rel, ab)
                H.check_against(*run_local(vals, rel, ab), ev, em, ("queue", n, name, G), vals)
        for name in ("d=31", "d=16", "cycle", "31,31"):
            vals = H.queue_rows(n, QUEUE_MANY[n], H.QUEUE_LAYOUTS[name], n)
            ev, em = OC.numeric(vals.view(np.float64), rel, ab)
            got = run_local(vals, rel, ab)
            H.check_against(*got, ev.view(np.uint64), em, ("queue, many tiles, C oracle", n, name))
            pick = np.random.default_rng(n).choice(len(vals), 3000, replace=False)
            bv, bm, _ = H.brute(vals[pick], rel, ab)
            H.check_against(got[0][pick], got[1][pick], bv, bm, ("queue, many tiles, brute force", n, name))
            assert len(np.unique(got[0])) == len(vals)
    assert_kernels_ran(prof, kernels(n, 161))


def _text(c):
    x = H.u2d(int(c))
    return "null" if (int(c) >> 32) == H.NONE_HI else repr(x)


def json_rows(n):
    """Family rows of 1 to 7 under the default tolerance, absent cells spelled None (a JSON record has every key), whose
    cells are all None or numbers whose repr the device path's to_double reads (it sends other numbers to the host), and
    whose brute-force value is finite or absent."""
    from tests.test_jsongpu_host_logic import parse_doubles
    vals = np.concatenate([H._rows(n, 0)[0], H._rows(n, 0, seed=1)[0]])
    vals = np.where((vals >> np.uint64(32)) == np.uint64(H.ABSENT_HI), np.uint64(H.NONE), vals)
    finite = [g for g, row in enumerate(vals)
              if all((int(c) >> 32) == H.NONE_HI or np.isfinite(H.u2d(int(c))) for c in row)]
    vals = vals[finite]
    texts = sorted({_text(c) for c in vals.reshape(-1)} - {"null"})
    _, ok = parse_doubles(texts)
    readable = {t for t, k in zip(texts, ok) if k}
    vals = vals[[g for g, row in enumerate(vals) if all(_text(c) in readable or _text(c) == "null" for c in row)]]
    ev, em, _ = H.brute(vals, *EDGE_EPS[0])
    keep = [g for g in range(len(vals)) if not (em[g] >> 27) & H.HAS or np.isfinite(H.u2d(int(ev[g])))]
    return vals[keep], ev[keep], em[keep]


@pytest.mark.parametrize("n", [2, 4, 8, 16, 32, 64])
def test_json_paths_on_the_edge_rows(n):
    """The finite / None family rows as {"x": <repr>} records: the device JSON path under JSON_DEVICE_ONLY takes every
    record (status 0), prints what its host instantiation with the C oracle prints and the brute force's value; H1 prints
    what it prints with the C oracle in K2's place.  No profiler session: the JSON paths launch from library threads."""
    _torch()
    from k_llms_b200 import _native as K
    vals, ev, em = json_rows(n)
    records = [['{"x": %s}' % _text(c) for c in row] for row in vals]
    blob, off, _ = K.pack_texts(records)
    res = K.consolidate_json_packed(blob, off, n, flags=K.JSON_DEVICE_ONLY)
    try:
        got, status = res.pairs(), list(res.status)
    finally:
        res.close()
    host, host_status = jsongpu_with_oracle(records)
    h1, h1_oracle = K.consolidate_json(records), consolidate_json_with_oracle(records)
    for r, texts in enumerate(records):
        assert status[r] == 0 and host_status[r] == 0 and got[r] == host[r], (n, r, texts, status[r], got[r], host[r])
        assert h1[r] is not None and h1[r] == h1_oracle[r], (n, r, texts, h1[r], h1_oracle[r])
        x = json.loads(got[r][0])["x"]
        if (int(em[r]) >> 27) & H.HAS:
            assert same(float(x), H.u2d(int(ev[r]))), (n, r, texts, got[r][0], H.u2d(int(ev[r])))
        else:
            assert x is None, (n, r, texts, got[r][0])
    print(f"\nn={n}: {len(records)} records")
    assert len(records) >= 150, len(records)
