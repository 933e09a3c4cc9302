"""Test helpers of the async dispatcher on the device JSON path (KC_JSON_NUMERIC_MEDOID): K5's oracle (numpy's own nanmean / argmax
on the reference's similarity matrix), a stand-in for the async entry's device call (the device phases on the host with the
oracles in the kernels' place), and the cell encoding of golden value groups."""
from __future__ import annotations

import json

import numpy as np

from oracle import columnar as OC
from tests.helpers import jsongpu_with_oracle

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


def oracle_native_consolidate(records, rel_eps, abs_eps, device=0, seq_logprobs=None, counts=None, flags=0):
    """consolidation._native_consolidate for the async dispatcher (flags = JSON_NUMERIC_MEDOID) with the device path's phases on
    the host and the oracle in the kernels' place."""
    from k_llms_b200 import _native as K
    assert flags == K.JSON_NUMERIC_MEDOID
    pairs, _ = jsongpu_with_oracle(records, seq_logprobs, flags=flags)
    if counts is not None:
        counts["device"] = counts.get("device", 0) + sum(p is not None for p in pairs)
    return pairs
