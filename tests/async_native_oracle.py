"""Test helpers of the async dispatcher on the device JSON path (KC_JSON_NUMERIC_MEDOID): K5's oracle (numpy's own nanmean / argmax
on the reference's similarity matrix), the device phases instantiated on the host with the oracles in the kernels' place, and the
cell encoding of golden value groups."""
from __future__ import annotations

import ctypes as c
import json

import numpy as np

from oracle import columnar as OC

GOLDEN = "tests/golden/async_numeric.json"


def golden_cases(kind: str):
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, GOLDEN)) as f:
        return [case for case in json.load(f)["cases"] if case["kind"] == kind]


def cells_of(groups, n: int) -> np.ndarray:
    """Value groups (lists of numbers / None, at most n each) -> K2's float64 [G, n] cells, absent-padded."""
    out = np.full((len(groups), n), OC.F64_ABSENT, dtype=np.float64)
    for g, vals in enumerate(groups):
        for i, v in enumerate(vals):
            out[g, i] = OC.F64_NONE if v is None else float(v)
    return out


def _isclose(a, b):
    """math.isclose(a, b, rel_tol=0.01) elementwise, as CPython computes it (math_isclose_impl): equal -> True, an infinity ->
    False, else |b - a| <= |0.01 * b| or <= |0.01 * a|, every operation one IEEE double operation."""
    with np.errstate(invalid="ignore", over="ignore"):
        diff = np.abs(b - a)
        close = (diff <= np.abs(0.01 * b)) | (diff <= np.abs(0.01 * a))
    return (a == b) | (~(np.isinf(a) | np.isinf(b)) & close)


def numeric_medoid(cells: np.ndarray, block: int = 2048):
    """K5's oracle: the reference's async numeric medoid (async_consensus_as_primitive, consensus_utils.py:1638-1688) on K2's
    cells float64 [G, n] (None / absent tags by their high word).  Over each group's k non-None cells: the k x k matrix of
    numerical_similarity (isclose -> 1.0, else 1e-8) with a NaN diagonal, np.nanmean of every row, np.argmax — numpy itself,
    on a stack of the groups with the same k.  Returns (best position among the non-None cells int32 [G], -1 for none; its
    mean float64 [G], NaN with fewer than two cells)."""
    cells = np.ascontiguousarray(cells, dtype=np.float64)
    G, n = cells.shape
    hi = (cells.view(np.uint64) >> np.uint64(32)).astype(np.uint32)
    live = (hi != np.uint32(OC.F64_NONE_BITS >> 32)) & (hi != np.uint32(OC.F64_ABSENT_BITS >> 32))
    k = live.sum(axis=1)
    best = np.where(k == 0, -1, 0).astype(np.int32)
    avg = np.full(G, np.nan)
    order = np.argsort(~live, axis=1, kind="stable")  # each row's live cells first, in candidate order
    for kk in np.unique(k[k >= 2]):
        idx = np.flatnonzero(k == kk)
        for s in range(0, len(idx), block):
            g = idx[s:s + block]
            x = np.take_along_axis(cells[g], order[g, :kk], axis=1)            # [B, kk]
            sims = np.where(_isclose(x[:, :, None], x[:, None, :]), 1.0, 1e-8)
            sims[:, np.arange(kk), np.arange(kk)] = np.nan
            means = np.nanmean(sims, axis=2)
            b = np.argmax(means, axis=1)
            best[g] = b
            avg[g] = means[np.arange(len(g)), b]
    return best, avg


def jsongpu_async_with_oracle(records, seq=None):
    """The device JSON path's phases under KC_JSON_NUMERIC_MEDOID, run on the host: kc_debug_jsongpu_plan_flags -> the C oracle
    in K1 (or K3b, seq float32 [R*n] given) and K4's place, numeric_medoid in K5's -> kc_debug_jsongpu_emit(_weighted).  Returns (pairs, status):
    pairs[r] = (content, likelihoods) or None where the device path declines the record (status[r] = its reason code)."""
    from k_llms_b200 import _native as K
    lib = K.load()
    R = len(records)
    if R == 0:
        return [], []
    blob, off, n = K.pack_texts(records, pinned=False)
    h = c.c_void_p()
    K.check(lib.kc_debug_jsongpu_plan_flags(blob.ctypes.data, off.ctypes.data, R, n, K.JSON_NUMERIC_MEDOID, c.byref(h)))
    try:
        vc, nc, st, gr = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        gv, gx = c.c_int64(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_inputs(h, c.byref(vc), c.byref(gv), c.byref(nc), c.byref(gx), c.byref(st)))
        K.check(lib.kc_debug_jsongpu_group_records(h, c.byref(gr)))
        vmeta, vweight = np.zeros(max(gv.value, 1), dtype=np.uint32), np.zeros(max(gv.value, 1), dtype=np.float32)
        if gv.value:
            codes = np.ctypeslib.as_array(c.cast(vc, c.POINTER(c.c_int8)), shape=(gv.value, n)).astype(np.int32)
            if seq is None:
                _, vmeta = OC.vote(codes, None)
            else:
                rec = np.ctypeslib.as_array(c.cast(gr, c.POINTER(c.c_int32)), shape=(gv.value,)).copy()
                _, vmeta, vweight = OC.weighted_vote(codes[:, None, :], np.asarray(seq, dtype=np.float32).reshape(R, n)[rec])
        best, avg = np.zeros(max(gx.value, 1), dtype=np.int32), np.zeros(max(gx.value, 1), dtype=np.float64)
        if gx.value:  # the oracle in K5's place
            best, avg = numeric_medoid(np.ctypeslib.as_array(c.cast(nc, c.POINTER(c.c_double)), shape=(gx.value, n)).copy())
        K.check(lib.kc_debug_jsongpu_set_numeric_medoid(h, best.ctypes.data, avg.ctypes.data))
        mc, so, go, gm = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_medoid_inputs(h, c.byref(mc), c.byref(so), c.byref(go), c.byref(gm)))
        midx, mavg = np.zeros(max(gm.value, 1), dtype=np.int32), np.zeros(max(gm.value, 1), dtype=np.float64)
        if gm.value:
            OC.lib().ko_medoid_str(mc, so, go, gm.value, midx.ctypes.data, mavg.ctypes.data)
        K.check(lib.kc_debug_jsongpu_set_medoid(h, midx.ctypes.data, mavg.ctypes.data))
        pc, po, pl, plo = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        K.check(lib.kc_debug_jsongpu_emit_weighted(h, vmeta.ctypes.data, vweight.ctypes.data if seq is not None else None, None, None,
                                                   c.byref(pc), c.byref(po), c.byref(pl), c.byref(plo)))
        status = np.ctypeslib.as_array(c.cast(st, c.POINTER(c.c_uint8)), shape=(R,)).copy()
        co = np.ctypeslib.as_array(c.cast(po, c.POINTER(c.c_int64)), shape=(R + 1,))
        lo = np.ctypeslib.as_array(c.cast(plo, c.POINTER(c.c_int64)), shape=(R + 1,))
        pairs = [None if status[r] else (c.string_at(pc.value + int(co[r]), int(co[r + 1] - co[r])).decode("ascii"),
                                         c.string_at(pl.value + int(lo[r]), int(lo[r + 1] - lo[r])).decode("ascii")) for r in range(R)]
        return pairs, list(status)
    finally:
        lib.kc_debug_jsongpu_free(h)


def oracle_native_consolidate(records, rel_eps, abs_eps, device=0, seq_logprobs=None, counts=None, flags=0):
    """consolidation._native_consolidate for the async dispatcher (flags = JSON_NUMERIC_MEDOID) with the device path's phases on
    the host and the oracle in the kernels' place."""
    from k_llms_b200 import _native as K
    assert flags == K.JSON_NUMERIC_MEDOID
    pairs, _ = jsongpu_async_with_oracle(records, seq_logprobs)
    if counts is not None:
        counts["device"] = counts.get("device", 0) + sum(p is not None for p in pairs)
    return pairs
