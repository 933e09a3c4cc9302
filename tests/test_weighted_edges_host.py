"""CPU: K3b's likelihood-weighted vote (DESIGN.md §5) at its decision edges, without a GPU.

The kernels that do not scan every class (weighted_core, wv_first_pass, wv_warp_walk in kc_extra.cuh) stop a walk once
wv_rest_bound(total, consumed) = (total - consumed) + kWvSlack * total falls below the best class weight.  This file
holds the edge families the GPU tests (tests/test_gpu_weighted_edges.py) run through every K3b kernel, a vectorised
brute force (every class summed in index order, no visiting order, no early stop), and a numpy restatement of
weighted_core's walk.  It checks the walk against the brute force over the families and a random sweep at n = 64, and
measures how much of kWvSlack the rounding of total, consumed and the class sums uses.

Every case is (codes int32 [R, F, n], seq_logprob float32 [R, n], none_code int32 [F] or None).  The logprobs come from a
search over float32 values with kexp, so the weights are exactly the ones a case needs: class sums that tie in fp32,
that flip between index-order fp32 summation and exact arithmetic, that sit within ulps of the stopping bound, or that
are clamped at kexp(-87)."""
import os
import re

import numpy as np
import pytest

from oracle import columnar as OC
from tests import weighted_oracle as W

F32 = np.float32
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "k_llms_b200", "csrc", "kc_extra.cuh")


def wv_slack() -> np.float32:
    """kWvSlack as kc_extra.cuh defines it, so these tests follow the constant."""
    m = re.search(r"constexpr\s+float\s+kWvSlack\s*=\s*([0-9.eE+-]+)f\s*;", open(HEADER).read())
    assert m, "kWvSlack not found in kc_extra.cuh"
    return F32(float(m.group(1)))


# ----------------------------------------------------------------------------- weights and the brute force, vectorised

def kexp_vec(x) -> np.ndarray:
    """kc::kexp elementwise (numpy rounds every float32 operation once and never fuses): bit-exact to W.kexp_np."""
    x = np.maximum(np.asarray(x, dtype=F32), F32(-87.0))
    t = x * F32(1.44269504)
    k = np.floor(t + F32(0.5))
    f = t - k
    p = np.full(f.shape, F32(0.00133336), dtype=F32)
    for c in (0.00961813, 0.05550411, 0.24022651, 0.69314718, 1.0):
        p = p * f + F32(c)
    return p * ((k.astype(np.int32) + 127) << 23).view(F32)


def weights(seq) -> np.ndarray:
    """[G, n] candidate weights kexp(s - max_k s_k) per row."""
    seq = np.asarray(seq, dtype=F32)
    return kexp_vec(seq - seq.max(axis=1, keepdims=True))


def map_cells(codes, nc):
    """The voting codes of raw cells: None votes as nc where nc >= 0; None without it and absent cells are -1."""
    codes = np.asarray(codes, dtype=np.int32)
    x = np.where(codes == -1, np.asarray(nc, dtype=np.int32)[:, None], codes)
    return np.where(x < -1, -1, x)


def pack_meta(idx, cnt, voters, present, flags):
    return ((idx & 0x3F) | ((cnt & 0x7F) << 6) | ((voters & 0x7F) << 13) | ((present & 0x7F) << 20)
            | ((flags & 0x1F) << 27)).astype(np.uint32)


def brute(codes, seq, nc=None):
    """The weighted vote of every group by enumerating all its classes: codes int [G, n] raw cells, seq float32 [G, n] the
    sums of each group's record, nc int [G] (None: no none_code).  Returns dict(win, meta, weight) and the internals the
    walk restatement and the reach counts reuse: x (voting codes), w, total, cw (class sums at each class's first index),
    first (first cell of a class)."""
    codes = np.asarray(codes, dtype=np.int32)
    G, n = codes.shape
    nc = np.full(G, -1, np.int32) if nc is None else np.asarray(nc, dtype=np.int32)
    x = map_cells(codes, nc)
    vote = x >= 0
    w = weights(seq)
    wv = np.where(vote, w, F32(0))  # adding +0.0 is exact: the index-order sums below skip non-voters
    total = np.zeros(G, F32)
    for i in range(n):
        total += wv[:, i]
    cw = np.zeros((G, n), F32)
    cnt = np.zeros((G, n), np.int32)
    later = np.zeros((G, n), bool)  # cell i has an earlier cell of its class
    ar = np.arange(n)
    for j in range(n):  # cw[:, i] = the weights of i's class in index order (cells before a class's first one add +0.0)
        m = vote & (x == x[:, j:j + 1]) & vote[:, j:j + 1]
        cw += np.where(m, wv[:, j:j + 1], F32(0))
        cnt += m
        later |= m & (ar > j)
    first = vote & ~later
    best_w = np.full(G, F32(-1))
    idx = np.zeros(G, np.int64)
    for i in range(n):  # first-seen order: a strictly heavier class replaces the best
        b = first[:, i] & (cw[:, i] > best_w)
        best_w = np.where(b, cw[:, i], best_w)
        idx = np.where(b, i, idx)
    rows = np.arange(G)
    tie = (first & (cw == best_w[:, None]) & (ar != idx[:, None])).any(axis=1)
    voters = vote.sum(axis=1)
    present = (codes >= -1).sum(axis=1)
    has = voters > 0
    idx = np.where(has, idx, 0)
    win = np.where(has, x[rows, idx], -1).astype(np.int32)
    with np.errstate(divide="ignore", invalid="ignore"):
        share = np.where(has, best_w / np.where(has, total, F32(1)), F32(0)).astype(F32)
    flags = np.where(has, 1 | np.where(tie, 4, 0), 0)
    meta = pack_meta(idx, np.where(has, cnt[rows, idx], 0), voters, present, flags)
    return dict(win=win, meta=meta, weight=share, x=x, w=w, total=total, cw=cw, first=first, vote=vote)


def flat(codes, seq, none_code):
    """[R, F, n] case -> per-group rows (codes [G, n], seq [G, n], nc [G])."""
    R, F, n = codes.shape
    nc = np.tile(none_code, R) if none_code is not None else np.full(R * F, -1, np.int32)
    return codes.reshape(R * F, n), np.repeat(seq, F, axis=0), nc


def first_pass(codes, seq, nc, ref, slack=None):
    """wv_first_pass's rule on the host: decided = the class of the record's heaviest candidate (first of the largest sums)
    holds cw_g > (total - cw_g) + total * kWvSlack in float32.  Returns the mask of groups with a voter it leaves to the walk."""
    slack = wv_slack() if slack is None else slack
    G, n = codes.shape
    imax = np.argmax(np.asarray(seq, dtype=F32), axis=1)
    graw = codes[np.arange(G), imax]
    guess = np.where(graw == -1, nc, graw)
    guess = np.where(guess < -1, -1, guess)
    m = (ref["x"] == guess[:, None]) & ref["vote"]
    cw_g = np.zeros(G, F32)
    for i in range(n):
        cw_g += np.where(m[:, i], ref["w"][:, i], F32(0))
    total = ref["total"]
    decided = (guess >= 0) & (cw_g > (total - cw_g) + total * slack)
    return ~decided & ref["vote"].any(axis=1)


def walk(codes, seq, nc, slack=None, bound_scale=F32(1)):
    """weighted_core's walk restated: visit the class of the heaviest waiting cell (first of equals), stop once
    wv_rest_bound(total, consumed) < best_w, an equally heavy class seen earlier takes the win.  Returns the results, the
    largest (unvisited class sum - (total - consumed)) / total seen at any stopping test, and per-group counts: swaps taken,
    and whether the answer differs from a walk that stopped one class early (groups that visited two classes or more)."""
    slack = wv_slack() if slack is None else slack
    ref = brute(codes, seq, nc)
    G, n = codes.shape
    x, vote, w, total, cw, first = ref["x"], ref["vote"], ref["w"], ref["total"], ref["cw"], ref["first"]
    rows = np.arange(G)
    ar = np.arange(n)
    wv = np.where(vote, w, F32(-1))
    c = np.where(vote.any(axis=1), x[rows, np.argmax(wv, axis=1)], -1)  # the heaviest voting cell's class (first of equals)
    live = vote.copy()
    best_w = np.full(G, F32(-1))
    best_idx = np.zeros(G, np.int64)
    best_cnt = np.zeros(G, np.int64)
    best_code = np.full(G, -1, np.int64)
    tie = np.zeros(G, bool)
    consumed = np.zeros(G, F32)
    prev = (best_code.copy(), best_idx.copy(), best_cnt.copy(), tie.copy())
    visits = np.zeros(G, np.int64)
    swaps = np.zeros(G, bool)
    margin = -np.inf
    active = live.any(axis=1)
    for _ in range(n + 1):
        active &= live.any(axis=1)
        rest = total - consumed
        waiting = first & live
        if (active & waiting.any(axis=1)).any():
            with np.errstate(divide="ignore", invalid="ignore"):
                over = (cw.astype(np.float64) - rest.astype(np.float64)[:, None]) / total.astype(np.float64)[:, None]
            margin = max(margin, float(np.where(waiting & active[:, None], over, -np.inf).max()))
        active &= ~(((rest + total * slack) * bound_scale) < best_w)
        if not active.any():
            break
        eq = (x == c[:, None]) & vote
        s = np.zeros(G, F32)
        for j in range(n):
            s += np.where(eq[:, j], w[:, j], F32(0))
        i = np.argmax(eq, axis=1)
        k = eq.sum(axis=1)
        prev = tuple(np.where(active, cur, p) for cur, p in zip((best_code, best_idx, best_cnt, tie), prev))
        gt = active & (s > best_w)
        same = active & ~gt & (s == best_w)
        sw = same & (i < best_idx)
        swaps |= sw
        take = gt | sw
        best_w = np.where(gt, s, best_w)
        best_idx = np.where(take, i, best_idx)
        best_cnt = np.where(take, k, best_cnt)
        best_code = np.where(take, c, best_code)
        tie = np.where(gt, False, tie | same)
        consumed = np.where(active, consumed + s, consumed)
        visits += active
        live &= ~(eq & active[:, None])
        wait = live & ~eq
        nwv = np.where(wait, w, F32(-1))
        c = np.where(active, np.where(wait.any(axis=1), x[rows, np.argmax(nwv, axis=1)], -1), c)
        active &= c >= 0
    voters = vote.sum(axis=1)
    present = (np.asarray(codes) >= -1).sum(axis=1)
    has = voters > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        share = np.where(has, best_w / np.where(has, total, F32(1)), F32(0)).astype(F32)
    meta = pack_meta(np.where(has, best_idx, 0), np.where(has, best_cnt, 0), voters, present,
                     np.where(has, 1 | np.where(tie, 4, 0), 0))
    differs = (visits >= 2) & ((prev[0] != best_code) | (prev[1] != best_idx) | (prev[2] != best_cnt) | (prev[3] != tie))
    return dict(win=np.where(has, best_code, -1).astype(np.int32), meta=meta, weight=share, margin=margin, swaps=swaps,
                early_differs=differs, ref=ref)


# ----------------------------------------------------------------------------- searching float32 logprobs for exact weights

def completion(partial, target):
    """All float32 s <= 0 whose weight w = kexp(s) gives float32(partial + w) == target exactly (empty if none)."""
    partial, target = F32(partial), F32(target)
    need = float(target) - float(partial)
    if not 0.0 < need <= 1.0 + 1e-6:
        return np.zeros(0, F32)
    s0 = F32(min(np.log(need), -1e-30))
    near = (s0.view(np.int32) + np.arange(-3000, 3001, dtype=np.int32)).view(F32)
    rel = (np.float64(s0) * (1.0 + np.linspace(-3e-3, 3e-3, 6001))).astype(F32)
    cand = np.unique(np.concatenate([near, rel, F32([0.0])]))
    cand = cand[np.isfinite(cand) & (cand <= 0)]
    return cand[(partial + kexp_vec(cand)) == target]


def class_logprobs(rng, m, target, tries=40):
    """m float32 logprobs whose weights, added in this order in float32 from +0.0, give exactly `target`; None if the
    search finds none."""
    target = F32(target)
    for _ in range(tries):
        s, acc = [], F32(0)
        for k in range(m - 1):
            want = (float(target) - float(acc)) * rng.uniform(0.3, 0.7) * (2.0 / (m - k))
            sk = F32(min(np.log(max(want, 1e-30)), 0.0))
            s.append(sk)
            acc = F32(acc + kexp_vec(sk))
        ok = completion(acc, target)
        if ok.size:
            return s + [F32(rng.choice(ok))]
    return None


_EXACT = {}


def exact_logprob(wt):
    """A float32 s with kexp(s) == wt exactly (wt a power of two here)."""
    if wt not in _EXACT:
        ok = completion(0.0, wt)
        assert ok.size, wt
        _EXACT[wt] = F32(ok[0])
    return _EXACT[wt]


# ----------------------------------------------------------------------------- the edge families
#
# A design is one record: labels [F, n] (class ids 0.., -1 = the cell does not vote) and seq [n] with max 0 (so the weights are
# kexp(s) exactly).  Structured designs give every field the same partition (make_case relabels it per field); partition-free
# ones (all weights near 1, clamped weights) draw a partition per field.

NOISE = (-30.0, -8.0)  # noise weights below 3.4e-4: 64 of them cannot outweigh a designed class


def _fill(rng, n, labels, seq, free, allvote, k0):
    """Noise in the positions `free`: non-voters, or light voters in 1-3 classes of their own (all voters when allvote)."""
    if not len(free):
        return
    if allvote or rng.random() < 0.5:
        kn = int(rng.integers(1, 4))
        labels[free] = k0 + rng.integers(0, kn, len(free))
        seq[free] = rng.uniform(*NOISE, len(free)).astype(F32)
    else:
        labels[free] = -1
        seq[free] = rng.uniform(-40.0, 0.0, len(free)).astype(F32) if rng.random() < 0.5 else F32(-5.0)


def _classes(rng, n, spec, allvote):
    """spec: list of (cells: list of s values in index order) per class, class 0 first.  Places them at random positions
    (each class's cells keep their index order), fills the rest with noise.  Returns labels [n], seq [n]."""
    need = sum(len(c) for c in spec)
    pos = rng.permutation(n)[:need]
    labels = np.full(n, -1, np.int64)
    seq = np.full(n, F32(-5.0), F32)
    k = 0
    for ci, cells in enumerate(spec):
        p = np.sort(pos[k:k + len(cells)])
        labels[p] = ci
        seq[p] = cells
        k += len(cells)
    _fill(rng, n, labels, seq, np.setdiff1d(np.arange(n), pos), allvote, len(spec))
    return labels, seq


def _lane_split(rng, n, labels, seq, a, b):
    """At n > 32, move cell a into lanes 0-31 and cell b into 32-63 (swapping contents), keeping the rest."""
    if n <= 32:
        return labels, seq
    pa, pb = int(rng.integers(0, 32)), int(rng.integers(32, n))
    for src, dst in ((a, pa), (b, pb)):
        if src != dst:
            labels[[src, dst]] = labels[[dst, src]]
            seq[[src, dst]] = seq[[dst, src]]
            if b == dst:
                b = src
    return labels, seq


def design_ties(rng, n, allvote=False):
    """Family 1: two or three classes of exactly equal fp32 weight; the record's heaviest cell (weight 1) in any of them,
    so the walk meets the first-seen class after a heavier cell's class and must swap."""
    if n < 2:
        return _classes(rng, n, [[F32(0)]], allvote)
    budget = n
    k = int(min(rng.choice([2, 3]), budget))
    sizes = [1] + [int(rng.integers(1, 4)) for _ in range(k - 1)]
    while sum(sizes) > budget:
        sizes[int(np.argmax(sizes))] -= 1
    sizes = [s for s in sizes if s > 0]
    low = rng.random() < 0.3 and not allvote and sum(sizes) < n  # the weight-1 cell does not vote: ties below it
    target = F32(rng.uniform(0.1, 0.9)) if low else F32(1.0)
    spec = []
    for m in sizes:
        cells = [F32(0)] * m if (m == 1 and target == 1) else class_logprobs(rng, m, target)
        if cells is None:
            cells = [F32(0)] if target == 1 else list(completion(0.0, target)[:1]) or [F32(0)]
        spec.append(list(cells) if m == len(cells) else [cells[0]])
    labels, seq = _classes(rng, n, spec, allvote)
    if low:
        free = np.flatnonzero(labels < 0)
        if len(free):
            seq[free[0]] = F32(0)
    if seq.max() < 0:
        seq[int(np.argmax(seq))] = F32(0)
    return labels, seq


def design_near(rng, n, allvote=False):
    """Family 2: A = [1, e, e(, e)] in some index order with e near half an ulp of A's partial sums, against B whose fp32 sum
    lies within two ulps of A's index-order fp32 sum or of A's exact sum: orders that flip between index-order fp32
    summation and exact arithmetic, pairs one ulp apart both ways."""
    m_a = int(min(n - 1, rng.integers(2, 5))) if n >= 3 else 1
    if m_a < 1:
        return design_ties(rng, n, allvote)
    e = [F32(np.log(2.0 ** -24 * rng.choice([0.5, 0.5, 0.75, 1.0, 1.5]) * rng.uniform(0.98, 1.02))) for _ in range(m_a - 1)]
    cells_a = [F32(0)] + e
    order = rng.permutation(m_a)
    cells_a = [cells_a[i] for i in order]
    acc = F32(0)
    for s in cells_a:
        acc = F32(acc + kexp_vec(s))
    exact = float(np.sum(kexp_vec(np.array(cells_a, F32)).astype(np.float64)))
    up, dn = np.nextafter(acc, F32(2)), np.nextafter(acc, F32(0))
    choices = [acc, up, dn, np.nextafter(up, F32(2)), np.nextafter(dn, F32(0)), F32(exact), np.nextafter(F32(exact), F32(2))]
    target = F32(choices[int(rng.integers(0, len(choices)))])
    m_b = int(min(n - m_a, rng.integers(2, 4)))
    spec = [cells_a]
    if m_b >= 1:
        cells_b = class_logprobs(rng, m_b, target) if target <= 1 or m_b >= 2 else None
        if cells_b is not None:
            spec.append(cells_b)
    if len(spec) > 1 and rng.random() < 0.5:
        spec = spec[::-1]
    return _classes(rng, n, spec, allvote)


def design_bound(rng, n, allvote=False):
    """Family 3: the stopping bound at its edge — the best class holds exactly half of the weight (dyadic weights, exact
    sums), the weight left after the first class equals it within a few ulps, or classes are visited in the order that
    shrinks the remainder slowest (single cells heaviest first, the winner a class of many light cells)."""
    v = int(rng.integers(0, 3))
    if v == 0 and n >= 3:  # H = 1 against dyadic classes that add up to exactly 1
        parts = [[0.5, 0.5], [0.5, 0.25, 0.25], [0.25, 0.25, 0.25, 0.25], [0.5, 0.25, 0.125, 0.125]][int(rng.integers(0, 4))]
        parts = parts[:n - 1] if sum(parts[:n - 1]) == 1.0 else [0.5, 0.5]
        spec = [[F32(0)]]
        if rng.random() < 0.5:  # as separate classes, or two of them in one class (still below H)
            spec += [[exact_logprob(p)] for p in parts]
        else:
            spec += [[exact_logprob(parts[0])], [exact_logprob(p) for p in parts[1:]]]
        return _classes(rng, n, spec, allvote)
    if v == 1 and n >= 3:  # H = 1, then one class (cells < 1) within a few ulps of it
        d = int(rng.integers(-3, 4))
        target = F32(1.0)
        for _ in range(abs(d)):
            target = np.nextafter(target, F32(2) if d > 0 else F32(0))
        m = int(min(n - 1, rng.integers(2, 5)))
        cells = class_logprobs(rng, m, target)
        if cells is not None:
            return _classes(rng, n, [[F32(0)], cells], allvote)
    # slowest shrink: k single cells 1 > w2 > ... then a class L of light cells that outweighs each of them
    k = max(1, min(8, n // 4))
    light = n - k
    if light < 2:
        return design_ties(rng, n, allvote)
    tops = [F32(0)] + [F32(np.log(1.0 - 0.04 * i)) for i in range(1, k)]
    lw = float(min(0.9 * (1.0 - 0.04 * (k - 1)), max(1.2 / light, 1e-3)))
    cells_l = list(np.full(light, F32(np.log(lw)), F32))
    labels = np.full(n, -1, np.int64)
    seq = np.full(n, F32(-5.0), F32)
    pos = rng.permutation(n)
    labels[pos[:k]] = np.arange(k)
    seq[pos[:k]] = tops
    labels[pos[k:]] = k
    seq[pos[k:]] = cells_l
    return labels, seq


def design_heavy(rng, n, allvote=False):
    """Family 4: the record's heaviest candidate — its cell does not vote (None / absent; make_case also spells it None with
    a none_code that votes), its class loses, or two candidates tie for the largest sum (at n > 32 one in lanes 0-31, one
    in 32-63)."""
    v = int(rng.integers(0, 3))
    if v == 0 and not allvote and n >= 2:
        k = int(rng.integers(2, 5))
        labels = rng.integers(0, k, n)
        seq = (-rng.exponential(1.5, n)).astype(F32)
        h = int(rng.integers(0, n))
        seq[h] = F32(0)
        labels[h] = -1
        return labels, seq
    if v == 1 and n >= 3:
        m = int(min(n - 1, rng.integers(2, 4)))
        cells = [F32(np.log(rng.uniform(0.55, 0.9))) for _ in range(m)]
        return _classes(rng, n, [[F32(0)], cells], allvote)
    k = int(rng.integers(1, 4))
    labels = rng.integers(0, k, n)
    seq = (-rng.exponential(1.0, n)).astype(F32)
    if n >= 2:
        a, b = rng.choice(n, 2, replace=False)
        a, b = min(a, b), max(a, b)
        seq[a] = seq[b] = F32(0)
        if rng.random() < 0.5:
            labels[b] = labels[a]
        labels, seq = _lane_split(rng, n, labels, seq, a, b)
    else:
        seq[0] = F32(0)
    return labels, seq


CLAMPED = F32([-86.9, -87.0, -87.1, -86.99, -87.01, -200.0, -1e4, -1e30])


def design_clamped(rng, n, allvote=False):
    """Family 5 (partition-free): gaps at -86.9, -87, -87.1 and far beyond, so weights clamp at kexp(-87) ~ 1.6e-38; the
    weight-1 cell does not vote in most records, leaving groups whose voters are all clamped (total ~ 1e-38)."""
    seq = CLAMPED[rng.integers(0, len(CLAMPED), n)].copy()
    h = int(rng.integers(0, n))
    seq[h] = F32(0)
    mute_h = not allvote and rng.random() < 0.7
    return None, seq, (h if mute_h else None)


def design_near_one(rng, n, allvote=False):
    """Family 3 (partition-free): every weight within a few ulps of 1, classes of equal sizes — the most rounding in total
    and consumed, class sums that differ only by it."""
    seq = (-rng.integers(0, 6, n) * 6e-8).astype(F32)
    seq[int(rng.integers(0, n))] = F32(0)
    return None, seq, None


FAMILIES = {1: [design_ties], 2: [design_near], 3: [design_bound, design_near_one], 4: [design_heavy], 5: [design_clamped]}
KNOCK = (None, 0, 31, 32, 63)  # family 6: one cell None or absent at these positions, or none


def _partition(rng, F, n, mute, allvote):
    k = int(rng.choice([2, 2, 3, 4]))
    if rng.random() < 0.5:  # classes of equal sizes
        labels = np.stack([rng.permutation(np.arange(n) % k) for _ in range(F)])
    else:
        labels = rng.integers(0, k, (F, n))
    if not allvote:
        labels[rng.random((F, n)) < 0.1] = -1
    if mute is not None:
        labels[:, mute] = -1
    return labels


def design_pool(rng, family, n, size=48):
    """`size` record designs of one family at n candidates: (labels [n] or None, seq [n], mute)."""
    allvote = family == 6
    makers = FAMILIES[family] if family != 6 else [design_ties, design_near, design_bound, design_near_one]
    out = []
    for i in range(size):
        d = makers[i % len(makers)](rng, n, allvote)
        if len(d) == 2:
            d = (d[0], d[1], None)
        if d[0] is not None:
            assert d[1].max() == 0, (family, d)
        out.append(d)
    return out


def make_case(rng, family, n, R, F, with_nc, pool=None):
    """One case of a family: R records of F fields at n candidates -> (codes int32 [R, F, n], seq float32 [R, n],
    none_code int32 [F] or None).  Every field relabels its record's classes with distinct codes in [0, 127] (int8 cells);
    with_nc gives fields a none_code that one class of the record uses (often the class of the heaviest candidate), whose
    cells are then spelled None — always the heaviest candidate's own cell."""
    pool = design_pool(rng, family, n) if pool is None else pool
    pick = rng.integers(0, len(pool), R)
    seq = np.stack([pool[i][1] for i in pick]).astype(F32)
    labels = np.empty((R, F, n), np.int64)
    for r, i in enumerate(pick):
        lab, _, mute = pool[i]
        labels[r] = np.broadcast_to(lab, (F, n)) if lab is not None else _partition(rng, F, n, mute, family == 6)
    if family == 6:  # the same rows with one cell knocked out at position 0, 31, 32 or 63 (field by field)
        for f in range(F):
            p = KNOCK[f % len(KNOCK)]
            if p is not None and p < n:
                labels[:, f, p] = -1
    hmax = np.argmax(seq, axis=1)
    none_code = None
    if with_nc:
        none_code = np.where(rng.random(F) < 0.7, rng.integers(0, 128, F), -1).astype(np.int32)
        none_code[0] = -1
    # per group: code = (a * label + b) mod 128, a odd (a bijection); b puts none_code on the chosen class
    a = 2 * rng.integers(0, 64, (R, F)) + 1
    b = rng.integers(0, 128, (R, F))
    if none_code is not None:
        h_lab = labels[np.arange(R), :, hmax]  # [R, F]
        k = labels.max(axis=2) + 1
        j = np.where((rng.random((R, F)) < 0.5) & (h_lab >= 0), h_lab, rng.integers(0, 64, (R, F)) % np.maximum(k, 1))
        b = np.where(none_code[None, :] >= 0, (none_code[None, :] - a * j) % 128, b)
    x = np.where(labels >= 0, (a[..., None] * labels + b[..., None]) % 128, -1)
    codes = x.astype(np.int32)
    nc_b = np.broadcast_to(none_code[None, :, None] if none_code is not None else np.full((1, F, 1), -1), codes.shape)
    is_h = np.arange(n)[None, None, :] == hmax[:, None, None]
    spell_none = (codes >= 0) & (codes == nc_b) & ((rng.random(codes.shape) < 0.5) | is_h)
    codes = np.where(spell_none, -1, codes)
    nonvote = labels < 0
    absent = nonvote & ((nc_b >= 0) | (rng.random(codes.shape) < 0.5))
    codes = np.where(nonvote, np.where(absent, -2, -1), codes).astype(np.int32)
    return np.ascontiguousarray(codes), np.ascontiguousarray(seq), none_code


def check_against(res, ref, what=""):
    """Winning code, every meta field (tie flag included) and the weight share's bits."""
    for k in ("win", "meta"):
        bad = np.flatnonzero(np.asarray(res[k]).astype(np.int64) != np.asarray(ref[k]).astype(np.int64))
        assert not bad.size, (what, k, bad[:10], np.asarray(res[k])[bad[:5]], np.asarray(ref[k])[bad[:5]])
    bad = np.flatnonzero(np.asarray(res["weight"], F32).view(np.uint32) != np.asarray(ref["weight"], F32).view(np.uint32))
    assert not bad.size, (what, "weight", bad[:10])


# ----------------------------------------------------------------------------- tests

def test_kexp_vec_is_bit_exact():
    xs = np.concatenate([np.linspace(-90, 0, 6001, dtype=F32), CLAMPED, F32([-0.0, -1e-30, -6e-8, -1.2e-7])])
    got = kexp_vec(xs)
    exp = np.array([W.kexp_np(x) for x in xs], F32)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


def test_slack_constant_is_read_from_the_header():
    assert F32(0) < wv_slack() < F32(1e-3)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8, 17, 32, 33, 64])
@pytest.mark.parametrize("family", [1, 2, 3, 4, 5, 6])
def test_brute_force_matches_restatement_and_c_oracle(family, n):
    """The vectorised brute force against W.brute_weighted_vote group by group (code, first index, share) and against the
    C oracle on every output, tie flag included."""
    rng = np.random.default_rng(1000 * family + n)
    for with_nc in (False, True):
        codes, seq, nc = make_case(rng, family, n, 120, 3, with_nc)
        ref = brute(*flat(codes, seq, nc))
        ew, em, ewt = OC.weighted_vote(codes, seq, nc)
        check_against(ref, dict(win=ew, meta=em, weight=ewt), (family, n, with_nc))
        c2, s2, nc2 = flat(codes, seq, nc)
        x = map_cells(c2, nc2)
        for g in range(0, len(c2), 7):
            code, first, share = W.brute_weighted_vote(np.where(x[g] >= 0, x[g], -1), s2[g])
            assert code == ref["win"][g] and F32(share).view(np.uint32) == ref["weight"][g].view(np.uint32), (g, family, n)
            if code >= 0:
                assert first == ref["meta"][g] & 0x3F


def _walk_families(rng, n, R=600, F=4):
    for family in (1, 2, 3, 4, 5, 6):
        for with_nc in (False, True):
            yield family, with_nc, make_case(rng, family, n, R, F, with_nc)


# families 1-3 must keep producing groups whose answer the last class the walk visits changes
EARLY_FLOOR = {1: 100, 2: 100, 3: 100}


@pytest.mark.parametrize("n", [2, 5, 8, 16, 32, 64])
def test_walk_equals_brute_force_and_slack_holds(n):
    """weighted_core's walk (heaviest waiting cell first, stop once wv_rest_bound < best_w, the swap) gives the brute force's
    answer on every family, and the rounding it has to absorb stays below kWvSlack."""
    slack = wv_slack()
    rng = np.random.default_rng(77 + n)
    worst = -np.inf
    early, swaps = {}, 0
    for family, with_nc, (codes, seq, nc) in _walk_families(rng, n):
        c2, s2, nc2 = flat(codes, seq, nc)
        got = walk(c2, s2, nc2, slack)
        check_against(got, got["ref"], (family, n, with_nc))
        worst = max(worst, got["margin"])
        early[family] = early.get(family, 0) + int(got["early_differs"].sum())
        swaps += int(got["swaps"].sum())
    print(f"\nn={n}: largest (unvisited class - (total - consumed)) / total = {worst:.3g} (kWvSlack {float(slack):.3g}); "
          f"groups the last visited class changes: {early}; swaps: {swaps}")
    assert worst < float(slack), f"rounding {worst:.3g} of total exceeds kWvSlack = {float(slack):.3g}"
    if n >= 8:
        for fam, floor in EARLY_FLOOR.items():
            assert early[fam] >= floor, (fam, early)
        assert swaps >= 50


def test_walk_random_sweep_n64_slack_margin():
    """A random sweep at n = 64 (few classes, skewed and flat logprobs, Nones) next to the families: the walk equals the
    brute force, and the largest rounding observed stays below kWvSlack with the margin reported."""
    slack = wv_slack()
    rng = np.random.default_rng(64064)
    G, n = 40000, 64
    codes = rng.integers(0, 4, (G, n)).astype(np.int32)
    codes[rng.random((G, n)) < 0.05] = -1
    kind = rng.integers(0, 3, G)[:, None]
    seq = np.where(kind == 0, -rng.exponential(0.3, (G, n)), np.where(kind == 1, -rng.integers(0, 3, (G, n)) * 6e-8,
                                                                      -rng.exponential(3.0, (G, n)))).astype(F32)
    seq[np.arange(G), np.argmax(seq, axis=1)] = F32(0)
    got = walk(codes, seq, np.full(G, -1, np.int32), slack)
    check_against(got, got["ref"], "sweep")
    worst = got["margin"]
    for family, with_nc, (c, s, nc) in _walk_families(rng, n, R=1000, F=2):
        g = walk(*flat(c, s, nc), slack)
        check_against(g, g["ref"], (family, with_nc))
        worst = max(worst, g["margin"])
    print(f"\nlargest (unvisited class - (total - consumed)) / total at n = 64: {worst:.3g}; kWvSlack = {float(slack):.3g}; "
          f"margin x{float(slack) / max(worst, 1e-30):.1f}")
    assert worst < float(slack), f"observed {worst:.3g} >= kWvSlack {float(slack):.3g} (margin {float(slack) - worst:.3g})"


def test_walk_without_slack_or_with_half_bound_goes_wrong():
    """The families reach what the slack protects: the restated walk with kWvSlack = 0 or with the bound halved gives wrong
    answers on them."""
    rng = np.random.default_rng(5)
    wrong = {}
    for slack in (F32(0), None):
        bad = 0
        for family, with_nc, (codes, seq, nc) in _walk_families(rng, 64, R=400, F=3):
            c2, s2, nc2 = flat(codes, seq, nc)
            got = walk(c2, s2, nc2, slack) if slack is not None else walk(c2, s2, nc2, bound_scale=F32(0.5))
            ref = got["ref"]
            bad += int(((got["win"] != ref["win"]) | (got["meta"] != ref["meta"])
                        | (got["weight"].view(np.uint32) != ref["weight"].view(np.uint32))).sum())
        wrong["no slack" if slack is not None else "half bound"] = bad
    assert wrong["no slack"] > 0 and wrong["half bound"] > 0, wrong

