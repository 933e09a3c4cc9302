"""Object-level oracle of the likelihood-weighted consensus (DESIGN.md §5, self-defined): the reference's client order
(oracle.consensus_py) with every vote leaf decided by the C oracle's K3b (ko_weighted_vote_i32) on cells kept at their
CANDIDATE's position — a candidate that is not a dict / list at some node is an absent cell below it.  Everything else
(dispatcher, parent_valid_frac, numeric clustering, medoid, key order) is oracle.consensus_py unchanged.

TEST INFRASTRUCTURE, used by tests/test_weighted_*.py only.
"""
from __future__ import annotations

from typing import Any, Callable, Optional, Sequence

import numpy as np

from oracle import columnar as OC
from oracle import consensus_py as O

NONE_CODE, ABSENT_CODE = -1, -2


def vote_cells(values: list, pos: Sequence[int], n: int, allow_none: bool):
    """The K1 / K3b cells of one vote leaf at candidate positions: (codes int32 [n], originals returned per cell)."""
    first = next(v for v in values if v is not None)
    codes = [ABSENT_CODE] * n
    table: dict = {}
    if isinstance(first, bool):  # cu:956: None and every falsy value vote False
        originals = [v or False for v in values]
        for p, k in zip(pos, originals):
            codes[p] = table.setdefault(k, len(table))
    else:
        originals = list(values)
        for p, v in zip(pos, values):
            if v is None and not allow_none:
                codes[p] = NONE_CODE
            else:
                codes[p] = table.setdefault(None if v is None else O.sanitize(v), len(table))
    return np.asarray(codes, dtype=np.int32), originals


def weighted_vote(values: list, pos: Sequence[int], seq: np.ndarray, settings, pvf: float):
    """One vote leaf: the heaviest class wins (ties: first seen), value = the first-seen original of the winning class,
    likelihood = round(pvf * float(weight), 5)."""
    n = len(seq)
    codes, originals = vote_cells(values, pos, n, settings.allow_none_as_candidate)
    win, meta, weight = OC.weighted_vote(codes.reshape(1, 1, n), np.asarray(seq, dtype=np.float32).reshape(1, n))
    f = OC.meta_fields(meta)
    assert int(f["flags"][0]) & 1, "a planned vote leaf has a voter"
    idx = int(f["idx"][0])
    return originals[list(pos).index(idx)], round(pvf * float(weight[0]), 5)


def consensus(values: list, seq: np.ndarray, settings=O.DEFAULTS, pvf: float = 1.0, embed: Optional[Callable] = None,
              pos: Optional[Sequence[int]] = None):
    """oracle.consensus_py.consensus with likelihood-weighted vote leaves; seq = the record's n candidate sums."""
    if pos is None:
        pos = list(range(len(values)))
    if not values:
        return None, pvf
    live = [v for v in values if v is not None]
    if not live:
        return None, 0.0
    head = live[0]
    if isinstance(head, (str, bool)) and all(len(str(v).strip().split()) < 3 for v in live):
        return weighted_vote(values, pos, seq, settings, pvf)
    if isinstance(head, dict):
        keep = [i for i, v in enumerate(values) if isinstance(v, dict)]
        dicts, sub_pos = [values[i] for i in keep], [pos[i] for i in keep]
        sub = pvf * (len(dicts) / len(values))
        keys: dict = {}
        for d in dicts:
            for k in d:
                keys.setdefault(k, None)
        out, conf = {}, {}
        for k in keys:
            if any(m in k for m in O.SKIPPED_KEY_MARKERS):
                continue
            out[k], conf[k] = consensus([d.get(k) for d in dicts], seq, settings, sub, embed, sub_pos)
        return out, conf
    if isinstance(head, list):
        keep = [i for i, v in enumerate(values) if isinstance(v, list)]
        lists, sub_pos = [values[i] for i in keep], [pos[i] for i in keep]
        sub = pvf * (len(lists) / len(values))
        longest = max(len(l) for l in lists)
        if longest == 0:
            return [], []
        out_l, conf_l = [], []
        for i in range(longest):
            v, c = consensus([l[i] if i < len(l) else None for l in lists], seq, settings, sub, embed, sub_pos)
            out_l.append(v)
            conf_l.append(c)
        return out_l, conf_l
    sub = pvf * (len(live) / len(values))
    return O.primitive(live, settings, sub, embed)


def client_order(values: list, seq: np.ndarray, settings=O.DEFAULTS, embed: Optional[Callable] = None, aligned: Any = None):
    """The client order (align, coerce to dicts, consensus) with weighted vote leaves.  aligned: the candidates after the
    alignment pre-pass when it is given (lists: the oracle restates only the dict part of the pre-pass)."""
    if aligned is None:
        aligned = [(d if isinstance(d, dict) else {}) for d in O.align_flat(values)] if len(values) >= 2 else values
    return consensus(aligned, seq, settings, 1.0, embed)


# ---- a pure numpy / float32 restatement of K3b for one group, to check the C oracle against

def _f32(x):
    return np.float32(x)


def kexp_np(x: np.float32) -> np.float32:
    x = _f32(x)
    if x < _f32(-87.0):
        x = _f32(-87.0)
    t = _f32(x * _f32(1.44269504))
    k = _f32(np.floor(_f32(t + _f32(0.5))))
    f = _f32(t - k)
    p = _f32(0.00133336)
    for c in (0.00961813, 0.05550411, 0.24022651, 0.69314718, 1.0):
        p = _f32(_f32(p * f) + _f32(c))
    scale = np.array([(int(k) + 127) << 23], dtype=np.int32).view(np.float32)[0]
    return _f32(p * scale)


def brute_weighted_vote(codes: Sequence[int], seq: Sequence[float]):
    """(winning code, first index of the winner, weight share float32) by enumerating the classes in first-seen order."""
    seq = [np.float32(s) for s in seq]
    smax = max(seq)
    w = [kexp_np(_f32(s - smax)) for s in seq]
    classes: dict = {}
    total = _f32(0.0)
    for i, c in enumerate(codes):
        if c < 0:
            continue
        total = _f32(total + w[i])
        if c not in classes:
            classes[c] = [i, _f32(0.0)]
        classes[c][1] = _f32(classes[c][1] + w[i])
    if not classes:
        return NONE_CODE, 0, _f32(0.0)
    best = None
    for c, (first, cw) in classes.items():  # first-seen order: a strictly heavier class replaces the best
        if best is None or cw > best[2]:
            best = (c, first, cw)
    return best[0], best[1], _f32(best[2] / total)
