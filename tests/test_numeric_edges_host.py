"""CPU: K2's numeric consensus (kc_numeric.cuh) at its decision edges, without a GPU.

K2 decides most groups through shortcuts whose boundaries decide the answer: the fast path's bitwise "at least half" guess
and strict-majority test, the certification of the nearest neighbours from their high words alone, the walk to at most two
extras and a numpy-order mean that assumes where each extra falls among the eight accumulators; the deferral queue; the
general core's 32-bit keys and low-bit repair, its three-compare chain test, its middle-element majority test, 64-bit
cluster masks and the tie order; and the n = 2 and n = 4 case analyses.  This file holds:
- edge families of groups built to land on those shortcuts (family 8: per-tile deferral layouts for the queue);
- `brute`, the numeric branch of the reference's consensus_as_primitive restated over K2's cell encoding, with numpy's own
  mean, median and std, checked against the C oracle and the object-level oracle;
- `kernel`, a restatement of K2's routing and arithmetic (numeric_pair, numeric_quad, numeric_fast_decide /
  numeric_fast_finish, numeric_core, numeric_tie) that reports which path every group takes, equals the brute force on every
  family, and goes wrong on the families under each of the MUTATIONS;
- host-counted floors on those paths, so that a generator change cannot quietly make the cases easy.
tests/test_gpu_numeric_edges.py runs the same families through every K2 kernel.

Rows are uint64 [G, n] cell bit patterns: finite values, None and absent (tagged by the high word alone), and any other
non-finite value (present, not None, not a number)."""
import collections
import math
import random
import struct

import numpy as np
import pytest

from oracle import columnar as OC
from oracle import consensus_py as O
from tests.helpers import EDGE_EPS, _down, _up

N_LIST = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64]
M32 = 0xFFFFFFFF
NONE_HI, ABSENT_HI = OC.F64_NONE_BITS >> 32, OC.F64_ABSENT_BITS >> 32
NONE, ABSENT = OC.F64_NONE_BITS, OC.F64_ABSENT_BITS
QNAN = 0x7FF8000000000000
HAS, SINGLE, TIE, NO_FINITE = 1, 2, 4, 8
BIAS = 0x00100000  # kFastBias
MAXF = 1.7976931348623157e308
LANES = (0, 31, 32, 63)
POW10 = [1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6]  # kPow10: 10.0 ** k, k = -6..6


def d2u(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def u2d(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def words(hi, lo):
    return u2d(((hi & M32) << 32) | (lo & M32))


def pack(idx, support, nn, present, flags):
    return (idx & 0x3F) | ((support & 0x7F) << 6) | ((nn & 0x7F) << 13) | ((present & 0x7F) << 20) | ((flags & 0x1F) << 27)


def pow2(n):
    p = 2
    while p < n:
        p *= 2
    return p


# non-finite cells that are not None or absent, and tags with other low words
ODD = [d2u(math.nan), d2u(-math.nan), d2u(math.inf), d2u(-math.inf), 0x7FFFFFFFFFFFFFFF, 0xFFF8000000000001, 0x7FF8C0E000000000,
       0x7FF0000000000001, 0x7FF8C0DD00000000]
TAGS = [NONE, ABSENT, NONE | 1, ABSENT | 0xFFFFFFFF]


# ----------------------------------------------------------------------------- the brute force

def _close(a, b, rel, ab):
    """cu:1134-1137 (the chain) and cu:1146-1148: |a - b| <= max(abs_eps, rel_eps * max(|a|, |b|, 1))."""
    return abs(a - b) <= max(ab, rel * max(abs(a), abs(b), 1.0))


def _close_pow10(a, b, rel, ab):
    """cu:1153-1160."""
    if a == 0.0 or b == 0.0:
        return _close(a, b, rel, ab)
    return any(_close(a, b * (10.0 ** k), rel, ab) for k in range(-6, 7))


def brute_group(cells, rel, ab):
    """One group: (value bits, result word, kind).  The census as kc_numeric_f64 documents it (absent cells are not in
    `values`, None cells are stripped by the dispatcher, any other non-finite cell counts in `total` and is not clustered),
    then cu:1098-1219 with none_count = 0."""
    present, live = 0, []
    for i, c in enumerate(cells):
        h = c >> 32
        if h == ABSENT_HI:
            continue
        present += 1
        if h != NONE_HI:
            live.append((i, c))
    total = len(live)
    if total == 0:
        return QNAN, pack(0, 0, 0, present, 0), "no value"
    if total == 1:  # cu:1085-1086: the object itself
        return live[0][1], pack(live[0][0], 1, 1, present, HAS | SINGLE), "single"
    xs = [x for x in (u2d(c) for _, c in live) if math.isfinite(x)]
    if not xs:
        return QNAN, pack(0, 0, total, present, NO_FINITE), "no finite"
    xs.sort()
    clusters = [[xs[0]]]
    for a, b in zip(xs, xs[1:]):
        if _close(a, b, rel, ab):
            clusters[-1].append(b)
        else:
            clusters.append([b])
    sizes = [len(c) for c in clusters]
    top = max(sizes)
    if top > total / 2 or sizes.count(top) == 1:
        return d2u(float(np.mean(clusters[int(np.argmax(sizes))]))), pack(0, top, total, present, HAS), \
            "majority" if top > total / 2 else "largest"
    centers = [float(np.median(c)) for c in clusters]
    spreads = [float(np.std(c)) if len(c) > 1 else 0.0 for c in clusters]
    supports = []
    for ci, c in enumerate(clusters):
        if len(c) != top:
            continue
        support = top
        for oi, other in enumerate(clusters):
            if oi != ci and len(other) < top and (
                    _close(centers[ci], centers[oi], rel, ab) or _close(abs(centers[ci]), abs(centers[oi]), rel, ab)
                    or _close_pow10(centers[ci], centers[oi], rel, ab)):
                support += len(other)
        supports.append((ci, support))
    supports.sort(key=lambda t: (-t[1], spreads[t[0]], -abs(centers[t[0]])))  # stable
    best, support = supports[0]
    return d2u(float(np.mean(clusters[best]))), pack(0, support, total, present, HAS | TIE), "tie"


def brute(vals, rel, ab):
    """(value uint64 [G], meta uint32 [G], kinds) of uint64 [G, n] rows."""
    with np.errstate(all="ignore"):
        out = [brute_group([int(c) for c in row], rel, ab) for row in np.asarray(vals, dtype=np.uint64)]
    return (np.array([o[0] for o in out], dtype=np.uint64), np.array([o[1] for o in out], dtype=np.uint32),
            [o[2] for o in out])


def nan_bits(u):
    u = np.asarray(u, dtype=np.uint64)
    return (((u >> np.uint64(52)) & np.uint64(0x7FF)) == np.uint64(0x7FF)) & ((u & np.uint64((1 << 52) - 1)) != np.uint64(0))


def check_against(got_value, got_meta, exp_value, exp_meta, what, rows=None):
    """Result words equal; values equal bit for bit, except that a NaN with no value only needs to be NaN on both sides."""
    gv, ev = np.asarray(got_value).view(np.uint64), np.asarray(exp_value).view(np.uint64)
    gm, em = np.asarray(got_meta).view(np.uint32), np.asarray(exp_meta).view(np.uint32)
    no_value = ((em >> 27) & HAS) == 0
    ok = (gm == em) & ((gv == ev) | (no_value & nan_bits(gv) & nan_bits(ev)))
    bad = np.flatnonzero(~ok)
    assert not bad.size, (what, bad.size, bad[:5], [hex(int(x)) for x in gv[bad[:3]]], [hex(int(x)) for x in ev[bad[:3]]],
                          OC.meta_fields(gm[bad[:3]]), OC.meta_fields(em[bad[:3]]),
                          None if rows is None else [[hex(int(c)) for c in rows[b]] for b in bad[:2]])


# ----------------------------------------------------------------------------- K2 restated

MUTATIONS = (
    "decide: 2c + nonfinite < N",       # numeric_fast_decide: <= -> <
    "decide: tagged > N - 1",           # numeric_fast_decide: > N - 2 -> > N - 1
    "certainly_far: d >= thr",          # d > thr -> d >= thr
    "certainly_far: magnitude (h, 0)",  # the above-side magnitude (h, -1) -> (h, 0)
    "walk: nb + na == 3",               # == 2u -> == 3u
    "finish: t == 1 ? l1",              # t == 1u ? l2 : v -> t == 1u ? l1 : v
    "far_bit: setp.lt",                 # the three setp.le -> setp.lt
    "core: 2 * (e0 - s0) >= m",         # > -> >=
    "core: repair skipped",
    "tie: olen > top",                  # olen >= top -> olen > top
    "tie: spread <=",                   # spread < best_spread -> <=
    "tie: |center| >=",                 # fabs(center) > fabs(best_center) -> >=
    "is_close_pow10: k < 12",           # k < 13 -> k < 12
    "np_mean16: len > 16",              # len >= 16 -> len > 16
    "pair: |c_hi| >=",                  # fabs(c_hi) > fabs(c_lo) -> >=
    "quad: sb <= sa",                   # sb < sa -> sb <= sa
    "quad: |mb| >=",                    # fabs(mb) > fabs(ma) -> >=
)
# A cell further into a high word above v is further from v by more than rel_eps times its extra magnitude (rel_eps < 1),
# so a cell that the true magnitude keeps uncertified but (h, 0) certifies far cannot be close: no output changes.
# A group with N - 1 tagged cells has them in more than half of its cells, so the guess takes their exponent and the group is
# deferred as "guess not finite" whatever the tagged test says.
UNCATCHABLE = ("certainly_far: magnitude (h, 0)", "decide: tagged > N - 1")


def dmax(a, b):
    return a if a > b else b


def is_close(a, b, rel, ab):
    return abs(a - b) <= dmax(ab, rel * dmax(dmax(abs(a), abs(b)), 1.0))


def pow10_k(a, b, rel, ab, mut):
    """is_close_pow10 past the plain test: the k of the first 10^k that makes a and b close, or None."""
    if a == 0.0 or b == 0.0:
        return None
    for k in range(12 if mut == "is_close_pow10: k < 12" else 13):
        if is_close(a, b * POW10[k], rel, ab):
            return k - 6
    return None


def far_bit(d, p, q, thr, mut):
    if mut == "far_bit: setp.lt":
        return not (d < p or d < q or d < thr)
    return not (d <= p or d <= q or d <= thr)


def np_sum(xs):
    """numpy's pairwise sum for n <= 128, seeded with +0.0 (np_sum)."""
    n = len(xs)
    if n < 8:
        res = -0.0
        for x in xs:
            res += x
    else:
        r = list(xs[:8])
        i, n8 = 8, n - n % 8
        while i < n8:
            for j in range(8):
                r[j] += xs[i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for x in xs[i:]:
            res += x
    return 0.0 + res


def np_mean(xs):
    return np_sum(xs) / len(xs)


def np_mean16(xs, mut):
    """np_mean16: predicated adds, the second round of accumulators only at len >= 16."""
    n = len(xs)
    if n < 8:
        return np_mean(xs)
    r = list(xs[:8])
    tail = 8
    if (n > 16) if mut == "np_mean16: len > 16" else (n >= 16):
        r = [r[j] + xs[8 + j] for j in range(8)]
        tail = 16
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for j in range(7):
        if tail + j < n:
            res += xs[tail + j]
    return (0.0 + res) / n


def np_median(xs):
    n = len(xs)
    if n & 1:
        return 0.0 + (-0.0 + xs[n // 2])
    return (0.0 + ((-0.0 + xs[n // 2 - 1]) + xs[n // 2])) / 2.0


def np_std(xs):
    mean = np_mean(xs)
    return math.sqrt(np_sum([(x - mean) * (x - mean) for x in xs]) / len(xs))


def core(cells, N, rel, ab, mut=None, info=None):
    """numeric_core<N> on N cells (a row padded with absent cells): census, 32-bit keys, the repair, the chain, the middle
    test, the cluster scan, np_mean16 / np_mean and numeric_tie."""
    info = {} if info is None else info
    thr = ab if ab > rel else rel
    IDX = N - 1
    hi = [c >> 32 for c in cells]
    present = sum(h != ABSENT_HI for h in hi)
    nn = sum(h != ABSENT_HI and h != NONE_HI for h in hi)
    m = sum((h & 0x7FF00000) != 0x7FF00000 for h in hi)
    if nn == 0:
        return QNAN, pack(0, 0, 0, present, 0)
    if nn == 1:
        idx = [i for i, h in enumerate(hi) if h != ABSENT_HI and h != NONE_HI][-1]
        return cells[idx], pack(idx, 1, 1, present, HAS | SINGLE)
    if m == 0:
        return QNAN, pack(0, 0, nn, present, NO_FINITE)
    keys = []
    for i, h in enumerate(hi):
        t = ((h ^ ((M32 if h >> 31 else 0) | 0x80000000)) - 0x00100000) & M32
        keys.append(((t | IDX) - (IDX - i)) & M32)
    keys.sort()
    xs = [u2d(cells[k & IDX]) for k in keys]
    if any(xs[k] < xs[k - 1] for k in range(1, N)):
        if any(xs[k] < xs[k - 1] for k in range(1, m)):
            info["repair"] = True
        if mut != "core: repair skipped":
            head = xs[:m]
            for i in range(1, m):  # insertion sort: equal values keep their places
                v, j = head[i], i - 1
                while j >= 0 and head[j] > v:
                    head[j + 1] = head[j]
                    j -= 1
                head[j + 1] = v
            xs[:m] = head
    starts, p_prev = 1, rel * xs[0]
    for k in range(1, N):
        p = rel * xs[k]
        if far_bit(xs[k] - xs[k - 1], p, -p_prev, thr, mut):
            starts |= 1 << k
        p_prev = p
    if m < N:
        starts &= (1 << m) - 1
    bounds = [k for k in range(N) if starts >> k & 1] + [m]
    clusters = [(s, e - s) for s, e in zip(bounds, bounds[1:])]
    c = m >> 1
    below = starts & ((2 << c) - 1)
    s0 = below.bit_length() - 1
    above = starts >> (c + 1)
    e0 = c + 1 + ((above & -above).bit_length() - 1) if above else m
    mid = 2 * (e0 - s0) >= m if mut == "core: 2 * (e0 - s0) >= m" else 2 * (e0 - s0) > m
    if mid:
        top, n_top, top_s = e0 - s0, 1, s0
        info["core"] = "middle"
    else:
        top = max(L for _, L in clusters)
        n_top = sum(L == top for _, L in clusters)
        top_s = next(s for s, L in clusters if L == top)
        info["core"] = "largest" if n_top == 1 else "tie"
    info["top start"] = top_s
    if n_top == 1:
        seg = xs[top_s:top_s + top]
        return d2u(np_mean16(seg, mut) if N <= 16 else np_mean(seg)), pack(0, top, nn, present, HAS)
    value, support = tie(xs, clusters, top, rel, ab, mut, info)
    return d2u(value), pack(0, support, nn, present, HAS | TIE)


def tie(xs, clusters, top, rel, ab, mut, info):
    """numeric_tie: for every cluster of the top size, the support strictly smaller clusters lend it (plain, signless or
    x 10^k), then the first strict improvement of (-support, spread, -|center|)."""
    best, cands = None, []
    for s, L in clusters:
        if L != top:
            continue
        center = np_median(xs[s:s + L])
        support = top
        for os_, OL in clusters:
            if (OL > top) if mut == "tie: olen > top" else (OL >= top):
                continue
            oc = np_median(xs[os_:os_ + OL])
            if is_close(center, oc, rel, ab):
                how = "plain"
            elif is_close(abs(center), abs(oc), rel, ab):
                how = "signless"
            else:
                k = pow10_k(center, oc, rel, ab, mut)
                how = None if k is None else f"x10^{k}"
            if how:
                support += OL
                info.setdefault("lent", set()).add(how)
        spread = np_std(xs[s:s + L]) if L > 1 else 0.0
        cands.append((s, support, spread, center))
        if best is None:
            better = True
        else:
            _, bsup, bspread, bcenter = best
            lt = spread <= bspread if mut == "tie: spread <=" else spread < bspread
            gt = abs(center) >= abs(bcenter) if mut == "tie: |center| >=" else abs(center) > abs(bcenter)
            better = support > bsup or (support == bsup and (lt or (spread == bspread and gt)))
        if better:
            best = (s, support, spread, center)
    s, support, spread, center = best
    peers = [cd for cd in cands if cd[0] != s]
    if all(p[1] < support for p in peers):
        info["tie"] = "support"
    elif all(p[2] > spread for p in peers if p[1] == support):
        info["tie"] = "spread"
    elif all(abs(p[3]) < abs(center) for p in peers if p[1] == support and p[2] == spread):
        info["tie"] = "|center|"
    else:
        info["tie"] = "order"
    if any(c[1] == support and c[2] == spread and abs(c[3]) == abs(center) for c in peers):
        info["|center| equal"] = True
    info["tie starts"] = [cd[0] for cd in cands]
    return np_mean(xs[s:s + top]), support


def numeric_pair(a, b, rel, ab, mut=None, info=None):
    """numeric_pair; info["pair"] names the outcome."""
    info = {} if info is None else info
    ah, bh = a >> 32, b >> 32
    a_abs, b_abs = ah == ABSENT_HI, bh == ABSENT_HI
    a_nn, b_nn = not a_abs and ah != NONE_HI, not b_abs and bh != NONE_HI
    a_fin = a_nn and (ah & 0x7FF00000) != 0x7FF00000
    b_fin = b_nn and (bh & 0x7FF00000) != 0x7FF00000
    present, nn = (not a_abs) + (not b_abs), a_nn + b_nn
    va, vb = u2d(a), u2d(b)
    if nn == 0:
        info["pair"] = "no value"
        return QNAN, pack(0, 0, 0, present, 0)
    if nn == 1:
        info["pair"] = "single"
        return (a if a_nn else b), pack(0 if a_nn else 1, 1, 1, present, HAS | SINGLE)
    if not a_fin and not b_fin:
        info["pair"] = "no finite"
        return QNAN, pack(0, 0, 2, present, NO_FINITE)
    if a_fin != b_fin:
        info["pair"] = "one finite"
        return d2u(0.0 + (-0.0 + (va if a_fin else vb))), pack(0, 1, 2, present, HAS)
    lo, hi = (vb, va) if va > vb else (va, vb)
    if is_close(lo, hi, rel, ab):
        info["pair"] = "close"
        return d2u((0.0 + ((-0.0 + lo) + hi)) / 2.0), pack(0, 2, 2, present, HAS)
    c_lo, c_hi = 0.0 + (-0.0 + lo), 0.0 + (-0.0 + hi)
    info["pair"] = "far, larger |hi|" if abs(c_hi) > abs(c_lo) else ("far, equal |.|" if abs(c_hi) == abs(c_lo) else "far, larger |lo|")
    take_hi = abs(c_hi) >= abs(c_lo) if mut == "pair: |c_hi| >=" else abs(c_hi) > abs(c_lo)
    return d2u(c_hi if take_hi else c_lo), pack(0, 1, 2, present, HAS | TIE)


def numeric_quad(w, rel, ab, mut=None, info=None):
    info = {} if info is None else info
    present = nn = m = first_nn = 0
    x = [0.0] * 4
    for i in (3, 2, 1, 0):
        h = w[i] >> 32
        absent, none, fin = h == ABSENT_HI, h == NONE_HI, (h & 0x7FF00000) != 0x7FF00000
        present += not absent
        if not absent and not none:
            nn += 1
            first_nn = i
        m += fin
        x[i] = u2d(w[i]) if fin else math.inf
    if nn == 0:
        return QNAN, pack(0, 0, 0, present, 0)
    if nn == 1:
        return w[first_nn], pack(first_nn, 1, 1, present, HAS | SINGLE)
    if m == 0:
        return QNAN, pack(0, 0, nn, present, NO_FINITE)

    def cex(i, j):
        if x[i] > x[j]:
            x[i], x[j] = x[j], x[i]
    cex(0, 1), cex(2, 3), cex(0, 2), cex(1, 3), cex(1, 2)
    b = [m > 1 and is_close(x[0], x[1], rel, ab), m > 2 and is_close(x[1], x[2], rel, ab), m > 3 and is_close(x[2], x[3], rel, ab)]
    info["quad bits"] = (m, tuple(b[:max(m - 1, 0)]))
    best_len = best_start = n_top = cur_len = cur_start = 0
    for i in range(4):
        joins = i > 0 and b[i - 1]
        cur_start = cur_start if joins else i
        cur_len = cur_len + 1 if joins else 1
        if i < m and (i + 1 == m or not b[min(i, 2)]):
            if cur_len > best_len:
                best_len, best_start, n_top = cur_len, cur_start, 1
            elif cur_len == best_len:
                n_top += 1

    def mean_of(s, z):
        acc = -0.0
        for i in range(s, s + z):
            acc += x[i]
        return (0.0 + acc) / z
    if n_top == 1:
        return d2u(mean_of(best_start, best_len)), pack(0, best_len, nn, present, HAS)
    if best_len == 1:
        best = 0.0 + (-0.0 + x[0])
        for i in range(1, 4):
            c = 0.0 + (-0.0 + x[i])
            if i < m and abs(c) > abs(best):
                best = c
        return d2u(best), pack(0, 1, nn, present, HAS | TIE)

    def stats(a, b_):
        mean = (0.0 + ((-0.0 + a) + b_)) / 2.0
        ta, tb = a - mean, b_ - mean
        return mean, math.sqrt((0.0 + ((-0.0 + ta * ta) + tb * tb)) / 2.0)
    ma, sa = stats(x[0], x[1])
    mb, sb = stats(x[2], x[3])
    lt = sb <= sa if mut == "quad: sb <= sa" else sb < sa
    gt = abs(mb) >= abs(ma) if mut == "quad: |mb| >=" else abs(mb) > abs(ma)
    info["quad pairs"] = "spread" if sb != sa else ("|center|" if abs(mb) != abs(ma) else "order")
    return d2u(mb if (lt or (sb == sa and gt)) else ma), pack(0, 2, nn, present, HAS | TIE)


def certainly_far(f, h, below, rel, thr, mut):
    if below:
        d, mag = f - words(h, M32), f
    else:
        d, mag = words(h, 0) - f, words(h, 0 if mut == "certainly_far: magnitude (h, 0)" else M32)
    return (d >= thr if mut == "certainly_far: d >= thr" else d > thr) and d > rel * mag


def fast_decide(cells, N, rel, thr, mut, info):
    """numeric_fast_decide<N>: None when the group is deferred (info['defer'] says why), else (v, e0, e1, word)."""
    hi = [c >> 32 for c in cells]
    lo = [c & M32 for c in cells]
    x = [(h + BIAS) & M32 for h in hi]
    top = max(hi)
    half = N // 2
    xv = sum(1 << b for b in range(32) if sum(xi >> b & 1 for xi in x) >= half)
    lv = sum(1 << b for b in range(32) if sum(li >> b & 1 for li in lo) >= half)
    nonfinite = sum(xi >> 31 for xi in x)
    below = max((xi - xv) & M32 for xi in x)
    above = min((xi - xv - 1) & M32 for xi in x)
    low_nf = min((xi + 0x80000000) & M32 for xi in x)
    c = sum(xi == xv for xi in x)
    bad = any(xi == xv and li != lv for xi, li in zip(x, lo))
    absent = sum(xi == ABSENT_HI + BIAS for xi in x) if top == ABSENT_HI else 0
    tagged = nonfinite
    no_majority = 2 * c + nonfinite < N if mut == "decide: 2c + nonfinite < N" else 2 * c + nonfinite <= N
    lone = tagged > N - 1 if mut == "decide: tagged > N - 1" else tagged > N - 2
    for cond, why in ((top > ABSENT_HI, "negative cell"), (xv >> 31, "guess not finite"), (bad, "shares v's high word"),
                      (no_majority, "no majority"), (lone, "single non-None cell"),
                      (nonfinite and low_nf < NONE_HI + BIAS - 0x80000000, "untagged non-finite")):
        if cond:
            info["defer"] = why
            return None
    hv = xv - BIAS
    v = words(hv, lv)
    hb, ha = (hv + below) & M32, (hv + above + 1) & M32
    has_b = below >= 0x80000000
    has_a = above < 0x7FFFFFFF and ha < 0x7FF00000
    need_b = has_b and not certainly_far(v, hb, True, rel, thr, mut)
    need_a = has_a and not certainly_far(v, ha, False, rel, thr, mut)
    word = (c << 6) + ((N - tagged) << 13) + ((N - absent) << 20) + (HAS << 27)
    e0 = e1 = v
    if N < 16:
        if need_b or need_a:
            info["defer"] = "close neighbour (n = 8)"
            return None
        return v, e0, e1, word
    xn, xa = (hb + BIAS if need_b else 0), (ha + BIAS if need_a else 0)
    if xn == 0:
        xn, xa = xa, 0
    while xn:
        nb, na = word & 3, (word >> 2) & 3
        if nb + na == (3 if mut == "walk: nb + na == 3" else 2):
            info["defer"] = "third extra"
            return None
        down = xn < xv
        sm = 0 if down else M32
        neg = (-(xn ^ sm)) & M32
        cnt, ln, beyond = 0, 0, 0
        for xi, li in zip(x, lo):
            beyond = max(beyond, ((xi ^ sm) + neg) & M32)
            if xi == xn:
                cnt += 1
                ln = li
        if cnt != 1:
            info["defer"] = "shares a neighbour's high word"
            return None
        e = words(xn - BIAS, ln)
        f = e0 if (nb if down else na) else v
        a, b = (e, f) if down else (f, e)
        close = not far_bit(b - a, rel * b, -(rel * a), thr, mut)
        side_done = not close
        if close:
            e1, e0 = e0, e
            word += 1 if down else 4
            hn = ((xn + beyond if down else xn - beyond) - BIAS) & M32
            exists = beyond >= 0x80000000 and (down or hn < 0x7FF00000)
            side_done = not exists or certainly_far(e, hn, down, rel, thr, mut)
            xn = (hn + BIAS) & M32
        else:
            info["uncertified far"] = info.get("uncertified far", 0) + 1
        if side_done:
            xn, xa = xa, 0
    return v, e0, e1, word


def fast_finish(d, N, mut):
    v, e0, e1, word = d
    c = (word >> 6) & 127
    if N < 16:
        res = -0.0
        if c >= 8:
            r = v
            for k in range(2, N // 8 + 1):
                if c >> 3 >= k:
                    r += v
            res = r * 8.0
        for k in range(1, 8):
            if c & 7 >= k:
                res += v
        return (0.0 + res) / c, word
    nb, na = word & 3, (word >> 2) & 3
    z, q, t = c + nb + na, (c + nb + na) >> 3, (c + nb + na) & 7
    f0 = v if nb == 0 else (e0 if na == 0 else e1)
    f1 = e1 if nb == 2 else v
    l2, l1 = (e1 if na == 2 else v), (v if na == 0 else e0)
    r0, r1, rp = f0, f1, -0.0
    for k in range(2, N // 8 + 1):
        if q >= k:
            r0 += v
            r1 += v
            rp += v
    r6 = rp + (l2 if t == 0 else v)
    r7 = rp + (l1 if t == 0 else ((l1 if mut == "finish: t == 1 ? l1" else l2) if t == 1 else v))
    r2 = rp + v
    s23 = r2 + r2
    tree = ((r0 + r1) + s23) + (s23 + (r6 + r7))
    small = z < 8
    sb, sa = (nb, na) if small else (0, min(na, t))
    sv = c if small else t - sa
    res = -0.0 if small else tree
    if sb >= 1:
        res += f0
    if sb >= 2:
        res += f1
    for k in range(1, 8):
        if sv >= k:
            res += v
    if sa >= 2:
        res += l2
    if sa >= 1:
        res += l1
    return (0.0 + res) / z, (word & ~15) + ((nb + na) << 6)


def kernel_group(cells, n, rel, ab, route="local", mut=None):
    """One group as kc_numeric_f64 (route 'local') or kc_numeric_f64_peers ('peers') computes it: (value bits, word, info)."""
    info = {}
    if route == "local" and n == 2:
        info["path"] = "pair"
        return (*numeric_pair(cells[0], cells[1], rel, ab, mut, info), info)
    if route == "local" and n == 4:
        info["path"] = "quad"
        return (*numeric_quad(cells, rel, ab, mut, info), info)
    thr = ab if ab > rel else rel
    if route == "local" and n in (8, 16, 32):
        d = fast_decide(cells, n, rel, thr, mut, info)
        if d is not None:
            value, word = fast_finish(d, n, mut)
            info["path"] = "fast"
            info["extras"] = (d[3] & 3, (d[3] >> 2) & 3)
            return d2u(value), word, info
        info["path"] = "deferred"
        return (*core(cells, n, rel, ab, mut, info), info)
    N = pow2(n)
    info["path"] = "core"
    return (*core(list(cells) + [ABSENT] * (N - n), N, rel, ab, mut, info), info)


def kernel(vals, rel, ab, route="local", mut=None):
    n = vals.shape[1]
    out = [kernel_group([int(c) for c in row], n, rel, ab, route, mut) for row in np.asarray(vals, dtype=np.uint64)]
    return (np.array([o[0] for o in out], dtype=np.uint64), np.array([o[1] for o in out], dtype=np.uint32),
            [o[2] for o in out])


# ----------------------------------------------------------------------------- building blocks of the families

def okey(x):
    u = d2u(x)
    return u if u < 1 << 63 else -(u - (1 << 63))


def from_okey(k):
    return u2d(k) if k >= 0 else u2d((-k) | (1 << 63))


def edge(v, rel, ab, side, close=None):
    """The farthest finite double on `side` (+1 above v, -1 below) that is still close to v (a transition point of the
    closeness test, by bisection over the ordered doubles); v itself when no other double is close."""
    close = close or (lambda e: _close(v, e, rel, ab))
    far = v + side * (abs(v) * 100.0 + ab * 100.0 + 100.0)
    far = max(-MAXF, min(MAXF, far)) if math.isfinite(far) else side * MAXF
    if close(far):
        return far
    lo, hi = okey(v), okey(far)
    while abs(hi - lo) > 1:
        mid = (lo + hi) // 2
        if close(from_okey(mid)):
            lo = mid
        else:
            hi = mid
    return from_okey(lo)


def tol(v, rel, ab):
    return max(ab, rel * max(abs(v), 1.0))


def messy(r, lo=1.0, hi=1000.0):
    """A value with a full, random mantissa."""
    return r.uniform(lo, hi) * 2.0 ** r.randint(-3, 3)


def fill(r, cells, n, tags_only=False):
    """cells plus None / absent (and, unless tags_only, other non-finite) cells up to n, shuffled; as bit patterns."""
    out = [c if isinstance(c, int) else d2u(c) for c in cells][:n]
    while len(out) < n:
        out.append(r.choice(TAGS) if tags_only or r.random() < 0.75 else r.choice(ODD))
    r.shuffle(out)
    return out


def far_values(r, v, k, rel, ab):
    """k finite values far from v and from each other (at least one tolerance apart under every EDGE_EPS)."""
    base = abs(v) if math.isfinite(v) and abs(v) < 1e300 else 1.0
    out, x = [], max(base, 1.0) * 37.0 + 50.0
    for _ in range(k):
        x = x * 13.0 if x < 1e290 else -(-x if x < 0 else x) / 1e10
        out.append(x if r.random() < 0.5 else -x)
    return out


def layout(r, sizes, rel, ab, sign=None):
    """Ascending values for clusters of the given sizes in that order: cluster bases 12x apart (far under every EDGE_EPS),
    members jittered inside the relative tolerance (identical copies when rel_eps is 0)."""
    out = []
    x0 = r.uniform(20.0, 30.0)
    neg = sign if sign is not None else r.random() < 0.3
    for j, s in enumerate(sizes):
        base = x0 * 12.0 ** j
        members = sorted(base * (1.0 + r.uniform(-1.0, 1.0) * rel * 0.2) if rel > 0 else base for _ in range(s))
        out += members
    return sorted(-x for x in out) if neg else out


# ----------------------------------------------------------------------------- the families

V_POOL = [0.0, -0.0, 5e-324, 2.0 ** -1022, 2.0 ** 52, 1e15 + 0.5, 1.7e308, 3.3, 1000.0, 0.1, 123456.0, 0.999999, 1.0]


def fam_census(r, n, rel, ab):
    """Family 1: c copies of v with 2c in {m - 1, m, m + 1, m + 2} (m finite cells) and the rest None, absent, NaN, +-inf and
    odd NaN payloads in each mix; N - 2 and N - 1 tagged cells; a single non-None cell (finite, NaN or inf) at lane 0, 31,
    32 or 63; no finite cell; every cell absent."""
    kind = r.randrange(10)
    v = r.choice(V_POOL)
    if kind >= 8 and n >= 2:  # exactly half v, half w with w's bits a subset of v's: the guess is v, 2c == m
        v = words(0x40000000 | r.getrandbits(20), r.getrandbits(32))
        w = words(d2u(v) >> 32 & ~0x00080000 & ~(1 << r.randrange(19)) & ~0x00100000, (d2u(v) & M32) & r.getrandbits(32))
        c = n // 2 + (kind == 9 and n % 2)
        return fill(r, [v] * c + [w] * (n - c), n, True)
    if kind <= 3:
        k_nf = min(n - 1, r.choice([0, 0, 1, 2, r.randint(0, n - 1)]))
        m = n - k_nf
        c = max(1, min(m, r.choice([m - 1, m, m + 1, m + 2]) // 2))
        rest = m - c
        if r.random() < 0.5:
            w = far_values(r, v, 1, rel, ab)[0]
            others = [w] * rest
        else:
            others = far_values(r, v, rest, rel, ab)
        tags_only = r.random() < 0.5
        cells = [v] * c + others
        out = fill(r, cells, n, tags_only)
        if not tags_only and k_nf:  # at least one non-finite cell that is not a tag
            i = r.choice([i for i, x in enumerate(out) if (x >> 32) in (NONE_HI, ABSENT_HI)] or [0])
            if (out[i] >> 32) in (NONE_HI, ABSENT_HI):
                out[i] = r.choice(ODD)
        return out
    if kind == 4:  # N - 2 or N - 1 tagged cells
        k = n - r.choice([1, 2]) if n >= 2 else n - 1
        cells = [v] * (n - k) if r.random() < 0.5 else far_values(r, v, n - k, rel, ab)
        return fill(r, cells, n, True)
    if kind == 5:  # a single non-None cell at a lane
        lanes = [i for i in LANES if i < n]
        lane = r.choice(lanes) if lanes and r.random() < 0.7 else r.randrange(n)
        out = [r.choice(TAGS) for _ in range(n)]
        out[lane] = d2u(v) if r.random() < 0.5 else r.choice(ODD)
        return out
    if kind == 6:  # no finite cell
        out = [r.choice(TAGS + ODD) for _ in range(n)]
        if n >= 2:
            for i in r.sample(range(n), 2):
                out[i] = r.choice(ODD)
        return out
    return [ABSENT] * n if r.random() < 0.5 else [r.choice(TAGS) for _ in range(n)]


NB_POOL = [1000.0, 123456.0, 1.0, 0.1, 0.5, 3.3, 1e15 + 0.5, 2.0 ** 52, 999999.0, 1e-7, 12.5, 40.0, 1.7e308, 5e-324]


def thr_pairs(rel, ab):
    """(v, e) with e exactly thr = max(abs_eps, rel_eps) from v and e at the end of its high word that certainly_far
    measures from ((h, 0) above v, (h, ~0) below), where thr rather than the relative term binds."""
    thr = ab if ab > rel else rel
    out = []
    if thr <= 0:
        return out
    for h in (0x3FF00000, 0x3FF80000, 0x40000000, 0x40080000, 0x40260000, 0x40340000, 0x3FE00000, 0x40590000):
        e = words(h, 0)
        v = e - thr
        if v >= 0 and e - v == thr:
            out.append((v, e))
        e = words(h, M32)
        v = e + thr
        if v - e == thr:
            out.append((v, e))
    return out


def fam_neighbours(r, n, rel, ab):
    """Family 2: a majority of v with one or two neighbours: at exactly the tolerance edge and 1 or 2 ulps inside or past
    it on either side (regimes where abs_eps, rel_eps * |v|, rel_eps * 1 or rel_eps * |e| binds); far cells that share
    the edge's high word (not certifiable from it) and cells in the next high word; two cells sharing a neighbour's high
    word, a cell sharing v's; a neighbour at the largest finite high word; negative cells and -0.0; a neighbour exactly
    thr from v at the end of its high word."""
    kind = r.randrange(9)
    v = r.choice(NB_POOL)
    if kind == 8:
        pairs = thr_pairs(rel, ab)
        if pairs:
            v, e = r.choice(pairs)
            ex = [e]
        else:
            kind = 0
    if kind <= 2:
        side = r.choice([1, -1])
        e = edge(v, rel, ab, side)
        k = r.choice([0, 0, 1, 2])
        e = (_up if (side > 0) == (r.random() < 0.5) else _down)(e, k) if k else e
        ex = [e] if kind < 2 else [e, edge(v, rel, ab, -side)]
    elif kind == 3:  # far, in the edge's high word (uncertifiable), or in the next high word (certifiable)
        side = r.choice([1, -1])
        e = edge(v, rel, ab, side)
        hh = d2u(e) >> 32
        cand = [_up(e, r.randint(1, 3)) if side > 0 else _down(e, r.randint(1, 3)),
                words(hh + side, 0 if side > 0 else M32), words(hh, M32 if side > 0 else 0)]
        ex = [c for c in cand if math.isfinite(c) and c != e][:r.randint(1, 2)]
    elif kind == 4:  # two cells share a neighbour's high word / one shares v's
        e = v + r.uniform(0.2, 0.8) * tol(v, rel, ab) * r.choice([1, -1])
        ex = [e, _up(e)] if r.random() < 0.5 else [r.choice([_up(v), _down(v), _up(v, 3)])]
    elif kind == 5:  # the largest finite high word
        v = words(0x7FEFFFFE, r.getrandbits(32))
        ex = [words(0x7FEFFFFF, r.getrandbits(32)), MAXF][:r.randint(1, 2)]
    elif kind == 6:  # negative cells, -0.0
        ex = [r.choice([-v if v else -5e-324, -0.0, -1.0])]
    elif kind == 7:  # the rel_eps * 1 and abs_eps regimes: |v| < 1
        v = r.choice([0.25, 1e-7, 5e-324, 0.0, 0.5])
        side = r.choice([1, -1])
        e = edge(v, rel, ab, side)
        ex = [e, _up(e)][:r.randint(1, 2)] if side > 0 else [e]
    ex = [x for x in ex if math.isfinite(x)]
    k_tag = r.randint(0, n // 3)
    m = n - k_tag
    c = max(1, m - len(ex) - r.choice([0, 0, 1]))
    return fill(r, [v] * c + ex + far_values(r, v, max(0, m - c - len(ex)), rel, ab), n, True)


def fam_extras(r, n, rel, ab):
    """Family 3: one and two extras in the splits (2, 0), (1, 1), (0, 2); a third close cell at either end; a cell close to
    an extra but far from v (the chain takes it); the cell beyond an extra exactly at, or one ulp past, its tolerance."""
    v = messy(r, 10.0, 5000.0)
    T = tol(v, rel, ab)
    split = r.choice([(1, 0), (0, 1), (2, 0), (1, 1), (0, 2)])
    ex, ends = [], {-1: v, 1: v}
    for side, count in ((-1, split[0]), (1, split[1])):
        for _ in range(count):
            f = ends[side]
            kind = r.random()
            if kind < 0.5:
                e = f + side * r.uniform(0.1, 0.9) * tol(f, rel, ab)
            elif kind < 0.8:  # close to the extra, far from v when it is the second one
                e = f + side * r.uniform(0.6, 0.99) * tol(f, rel, ab)
            else:
                e = edge(f, rel, ab, side)
            ex.append(e)
            ends[side] = e
    kind = r.randrange(4)
    if kind == 0:  # a third close cell at either end
        side = r.choice([-1, 1])
        ex.append(ends[side] + side * r.uniform(0.1, 0.5) * tol(ends[side], rel, ab))
    elif kind == 1:  # the cell beyond the outermost extra: at its edge or one ulp past it
        side = -1 if split[0] and (not split[1] or r.random() < 0.5) else 1
        e = edge(ends[side], rel, ab, side)
        ex.append(e if r.random() < 0.5 else (_up(e) if side > 0 else _down(e)))
    elif kind == 2:
        ex.append(v + r.choice([-1, 1]) * T * r.uniform(2.5, 4.0))
    m = n - r.randint(0, n // 4)
    c = max(1, m - len(ex))
    return fill(r, [v] * c + ex, n, True)


def alternative_means(cl, nb, na):
    """The means a kernel could wrongly compute for the sorted cluster cl, as tuples: a numpy mean must differ from at least
    one mean of each.  A left-to-right sum; numpy's order with every cell one accumulator over, either way, which moves each
    extra into a neighbouring accumulator or between an accumulator and the tail (with two extras); eight equal
    accumulators (8 * r, r the sum in accumulator 2, which holds copies only) plus the tail (when an extra is in an
    accumulator)."""
    z = len(cl)
    s = -0.0
    for x in cl:
        s += x
    alts = [((0.0 + s) / z,)]
    # With one extra the other accumulators hold equal sums, so where the extra sits cannot change the bits; with two, one
    # of the two placements is enough (some only swap two accumulators that are added to each other first).
    if nb + na == 2:
        alts.append((float(np.mean(np.roll(cl, 1))), float(np.mean(np.roll(cl, -1)))))
    if z >= 16 and (nb or na > z % 8):  # some extra inside the accumulators (extras in the tail leave 8 * r exact)
        r_ = -0.0
        for x in cl[2:z - z % 8:8]:
            r_ += x
        tail = r_ * 8.0
        for x in cl[z - z % 8:]:
            tail += x
        alts.append(((0.0 + tail) / z,))
    return alts


def sum_order_cases(r, n, rel, ab, tries=60):
    """Family 4, found by search: for every (z, nb, na) with 8 <= z <= n, clusters of z = c + nb + na values (c copies of v
    and nb extras below it, na above) whose numpy mean has other bits than each alternative_means; smaller clusters too."""
    out = []
    splits = [(0, 0), (1, 0), (0, 1), (2, 0), (1, 1), (0, 2)] if rel >= 0.01 else [(0, 0)]
    for z in range(2, n + 1):
        for nb, na in splits:
            c = z - nb - na
            if c < 1:
                continue
            for _ in range(tries if z >= 8 else 1):
                v = messy(r)
                T = tol(v, rel, ab)
                below = sorted(v - r.uniform(0.05, 0.45) * T for _ in range(nb))
                above = sorted(v + r.uniform(0.05, 0.45) * T for _ in range(na))
                hs = [d2u(x) >> 32 for x in below + above + [v]]
                if len(set(hs)) != len(hs):
                    continue
                cl = below + [v] * c + above
                mean = float(np.mean(cl))
                if z < 8 or all(any(d2u(a) != d2u(mean) for a in alt) for alt in alternative_means(cl, nb, na)):
                    out.append((z, nb, na, v, below + above))
                    break
    return out


def fam_general(r, n, rel, ab):
    """Family 5: low-bit repair (high words that differ only in the low log2 N bits, or only low words, descending with the
    index); chain edges a < 0 < b with |a|, |b| < 1; -1.7e308 next to 1.7e308; a cluster of 2 * len in {m, m + 1} that starts
    or ends at the middle element; at n = 64 clusters starting at 31, 32 or 33 and ties on both sides of mask bit 32."""
    N = pow2(n)
    kind = r.choice([0, 1, 2, 3, 4, 4, 4]) if n == 64 else r.randrange(4)
    if kind == 0:
        k = r.randint(2, n)
        h = (r.choice([0x3FF00000, 0x40A00000, 0x00100000]) + r.getrandbits(19)) & ~(N - 1)
        if r.random() < 0.5:
            vals = sorted((words(h + r.randrange(N), r.getrandbits(32)) for _ in range(k)), reverse=True)
        else:
            vals = sorted((words(h, r.getrandbits(32)) for _ in range(k)), reverse=True)
        if r.random() < 0.3:
            vals = [-x for x in vals][::-1]
        pos = sorted(r.sample(range(n), k))
        out = [r.choice(TAGS) for _ in range(n)]
        for p, x in zip(pos, vals):
            out[p] = d2u(x)
        return out
    if kind == 1:  # a < 0 < b, |a|, |b| < 1: at the chain's edge where the tolerance near zero is below 1, else close or far
        T = tol(0.0, rel, ab)
        if 0 < T < 1:
            a = -r.uniform(0.05, 0.95) * T
            b = edge(a, rel, ab, 1)
            b = r.choice([b, _up(b), _down(b)])
        else:
            a, b = -r.uniform(0.05, 0.95), r.uniform(0.05, 0.95)
        ka = r.randint(1, max(1, n // 2))
        return fill(r, [a] * ka + [b] * max(1, n - ka - r.randint(0, 2)), n, True)
    if kind == 2:
        cells = [-1.7e308, 1.7e308, -MAXF, MAXF][:r.randint(2, 4)]
        return fill(r, cells * max(1, n // 4), n, True)
    # a cluster whose 2 * len is m or m + 1, starting or ending at the middle element c = m >> 1
    m = r.randint(2, n) if kind == 3 else n - r.randint(0, 2)
    if kind == 3:
        L = (m + r.randint(0, 1)) // 2
        L = max(1, min(L, m))
        c = m >> 1
        s = c if r.random() < 0.5 else max(0, c - L + 1)
        s = min(s, m - L)
        rest_lo, rest_hi = s, m - s - L
        groups = [1] * rest_lo + [L] + [1] * rest_hi
        if 2 * L == m and r.random() < 0.5:  # the other half as one cluster: a tie
            groups = ([L, rest_hi] if rest_hi else [rest_lo, L]) if rest_lo == 0 or rest_hi == 0 else groups
            groups = [g for g in groups if g]
    else:  # n = 64: clusters starting at 31, 32, 33, and equal clusters on both sides of bit 32
        s = r.choice([31, 32, 33])
        L = r.randint(2, min(16, m - s))
        if r.random() < 0.5:
            groups = [1] * (s - L) + [L] + [L] + [1] * (m - s - L) if s >= L else [1] * s + [L] + [1] * (m - s - L)
        else:
            groups = [1] * s + [L] + [1] * (m - s - L)
        groups = [g for g in groups if g > 0]
    vals = layout(r, groups, rel, ab)
    return fill(r, vals, n, True)


def fam_ties(r, n, rel, ab):
    """Family 6: 2 to 8 tied clusters of even or odd size; support lent through the plain, the signless and the x 10^k test
    (k in -6..6, at the tolerance edge after the multiplication, one ulp inside or past it); zero centers; equal supports
    with equal spreads or spreads one ulp apart, then equal |centers| (-x and x: the lower one wins) or one ulp apart."""
    kind = r.randrange(4)
    if kind == 0:  # k tied clusters of s, lenders of smaller size
        s = r.choice([1, 2, 3, 4])
        k = max(2, min(r.randint(2, 8), n // max(s, 1)))
        if k * s > n:
            return fam_general(r, n, rel, ab)
        cl = layout(r, [s] * k, rel, ab)
        return fill(r, cl + far_values(r, cl[0], r.randint(0, n - k * s), rel, ab)[:1], n, True)
    if kind == 1:  # a lender through -x or x * 10^-k
        return lender_row(r, n, rel, ab, r.choice(["signless"] + LENDER_KS + [-6, 6, -6, 6]))
    if kind == 2:  # equal spreads and |centers|: [-x - d, -x + d] and [x - d, x + d], dyadic; one-ulp variants
        s = 2
        if 2 * s > n:
            return fam_pair_table(r, n, rel, ab) if n == 2 else fill(r, [1.0, -1.0], n, True)
        x = float(r.choice([100.0, 6.5, 1024.0, 48.25, 3000.0]))
        d = x * rel * 0.25 if rel > 0 else 0.0
        d = float(np.float64(d).round(0)) / 2.0 ** 4 if d > 1 else 2.0 ** -6 * (rel > 0)
        a = [-x - d, -x + d]
        b = [x - d, x + d]
        var = r.randrange(5)
        if var == 1:
            b = [_up(b[0]), _up(b[1])]          # |center| one ulp larger
        elif var == 2:
            b = [b[0], _up(b[1])]              # spread (and center) a little larger
        elif var == 3:
            a = [a[0], _up(a[1])]
        elif var == 4:
            b = [_up(x), _up(x)] if d == 0 else b
        k = r.choice([2, 2, 3])
        extra = [0.0, 0.0] if k == 3 and n >= 6 else []
        return fill(r, a + b + extra, n, True)
    # zero centers
    cells = [r.choice([[0.0, -0.0], [0.0, 0.0], [-0.0, -0.0]])] + [[x, x] for x in (1.0, -1.0, 5e-324)]
    flat = [c for pair in cells[:max(2, n // 2)] for c in pair]
    return fill(r, flat, n, True)


LENDER_KS = [k for k in range(-6, 7) if k]  # k = 0 is the plain test


def lender_row(r, n, rel, ab, how):
    """Two tied clusters of s in {2, 3} and a smaller cluster whose center lends one of them support: through the signless
    test (how == "signless": about -center) or the x 10^k test (how == k: at the edge of closeness to center / 10^k after
    the multiplication, or one ulp inside or past it)."""
    s = r.choice([2, 3])
    if 2 * s + 1 > n:
        return fam_pair_table(r, n, rel, ab) if n == 2 else fill(r, [1.0, -1.0], n, True)
    cl = layout(r, [s, s], rel, ab, sign=False)
    centre_cluster = cl[:s] if r.random() < 0.5 else cl[s:]
    center = float(np.median(centre_cluster))
    if how == "signless":
        o = -center * (1.0 + r.uniform(-0.5, 0.5) * rel)
    else:
        o0 = center / (10.0 ** how)
        o = edge(o0, rel, ab, r.choice([1, -1]), close=lambda e: _close(center, e * (10.0 ** how), rel, ab))
        o = r.choice([o, o, _up(o), _down(o)])
    return fill(r, cl + [o] * r.randint(1, s - 1), n, True)


def fam_pair_table(r, n, rel, ab):
    """Family 7 at n = 2: every outcome of numeric_pair; elsewhere a pair padded with tags."""
    v = r.choice(NB_POOL[:-2])
    kind = r.randrange(7)
    if kind == 0:
        cells = [r.choice(TAGS), r.choice(TAGS)]
    elif kind == 1:
        cells = [r.choice([d2u(v), r.choice(ODD)]), r.choice(TAGS)]
    elif kind == 2:
        cells = [r.choice(ODD), r.choice(ODD)]
    elif kind == 3:
        cells = [d2u(v), r.choice(ODD)]
    elif kind == 4:
        e = edge(v, rel, ab, r.choice([1, -1]))
        cells = [d2u(v), d2u(r.choice([e, _up(e), _down(e), v]))]
    elif kind == 5:
        cells = [d2u(v), d2u(-v)]
    else:
        cells = [d2u(v), d2u(far_values(r, v, 1, rel, ab)[0])]
    r.shuffle(cells)
    return fill(r, cells, n, True) if n != 2 else cells


def fam_quad_table(r, n, rel, ab):
    """Family 7 at n = 4: every close-bit pattern of numeric_quad for m = 1..4 finite cells with the non-finite cells in
    every position; two pairs with equal spreads and +-|centers|."""
    m = r.randint(1, 4)
    pattern = r.getrandbits(max(m - 1, 0)) if m > 1 else 0
    x = r.choice([1.0, 10.0, 250.0, -400.0, 0.3])
    vals = [x]
    for i in range(m - 1):
        if pattern >> i & 1:
            x = x + abs(x) * rel * 0.3 if rel > 0 else x
        else:
            x = x + abs(x) * 20.0 + 20.0
        vals.append(x)
    if m == 4 and r.random() < 0.3:
        y = r.choice([100.0, 7.0])
        d = 2.0 ** -4 if rel > 0 else 0.0
        vals = [-y - d, -y + d, y - d, y + d] if r.random() < 0.6 else [-y, -y, y, y]
    out = [d2u(v) for v in vals] + [r.choice(TAGS + ODD) for _ in range(4 - m)]
    r.shuffle(out)
    return out if n == 4 else fill(r, out, n, True)


def fam_tables(r, n, rel, ab):
    return fam_pair_table(r, n, rel, ab) if n == 2 else fam_quad_table(r, n, rel, ab)


def sum_order_row(r, n, case, rel, ab):
    """A sum_order_cases cluster in n cells.  The other cells are None and absent tags, and up to nb + na of them +0.0 (a
    far cluster without a set bit) when it is far from v: with c = n / 2 copies of v the fast path's "at least half" guess is
    then still v, since no bit outside v's can be set in half of the cells."""
    z, nb, na, v, ex = case
    cells = [v] * (z - nb - na) + ex
    if z < n and not _close(0.0, min(cells), rel, ab):
        cells += [0.0] * min(n - z, max(1, nb + na))
    out = [d2u(x) for x in cells] + [r.choice([NONE, ABSENT]) for _ in range(n - len(cells))]
    r.shuffle(out)
    return out


def sum_order_rows(n, eps_i, seed=0):
    """Family 4 in full: every sum_order_cases cluster at n under EDGE_EPS[eps_i], one row each."""
    rel, ab = EDGE_EPS[eps_i]
    r = random.Random(9100 + 31 * n + 7 * eps_i + seed)
    cases = sum_order_cases(r, n, rel, ab)
    return np.array([sum_order_row(r, n, c, rel, ab) for c in cases], dtype=np.uint64).reshape(len(cases), n), cases


def fam_sum_order(r, n, rel, ab, cases):
    return sum_order_row(r, n, r.choice(cases), rel, ab)


MAKERS = {1: fam_census, 2: fam_neighbours, 3: fam_extras, 5: fam_general, 6: fam_ties, 7: fam_tables}
FAMILIES = (1, 2, 3, 4, 5, 6, 7)


def families_for(n):
    return [f for f in FAMILIES if not (f == 7 and n not in (2, 4)) and not (f in (3, 4, 5, 6) and n < 2)]


def family_rows(seed, n, rel, ab, per_family):
    """per_family rows of every family that applies at n, family after family: (uint64 [G, n], family [G])."""
    r = random.Random(seed)
    rows, fam = [], []
    cases = sum_order_cases(random.Random(seed + 1), n, rel, ab) if n >= 2 else []
    for f in families_for(n):
        for j in range(per_family):
            if f == 4:
                row = fam_sum_order(r, n, rel, ab, cases)
            elif f == 6 and j % 3 == 0:  # every x 10^k lender and the signless one in turn
                row = lender_row(r, n, rel, ab, (LENDER_KS + ["signless"])[(j // 3) % (len(LENDER_KS) + 1)])
            else:
                row = MAKERS[f](r, n, rel, ab)
            assert len(row) == n, (f, n)
            rows.append(row)
            fam.append(f)
    return np.array(rows, dtype=np.uint64).reshape(len(rows), n), np.array(fam)


# ----------------------------------------------------------------------------- family 8: queue layouts

QUEUE_D = (0, 1, 2, 16, 31, 32)
QUEUE_LAYOUTS = {"d=%d" % d: (d,) for d in QUEUE_D}
QUEUE_LAYOUTS.update({"cycle": QUEUE_D, "16,16": (16, 16), "31,31": (31, 31), "1,31": (1, 31)})


def queue_rows(n, G, layout_d, seed):
    """Family 8: G groups, tile t (groups 32t .. 32t + 31) with layout_d[t % len] deferred groups at random lanes.  A decided
    group is n - 1 copies of a value of its own and a None; a deferred one is that value and -64 times it in halves (no
    majority, and a negative cell).  Every group's result is distinct, so that a result stored at another index shows."""
    rng = np.random.default_rng(seed)
    tiles = -(-G // 32)
    d = np.array([layout_d[t % len(layout_d)] for t in range(tiles)])
    lane_rank = np.argsort(rng.random((tiles, 32)), axis=1)  # a random order of the lanes per tile
    defer = (lane_rank < d[:, None]).reshape(-1)[:G]
    v = 1000.0 + np.arange(G) * 0.5 + 0.25
    cells = np.repeat(v[:, None], n, axis=1)
    cells[~defer, n - 1] = OC.F64_NONE
    cells[defer, n // 2:] = -64.0 * v[defer, None]
    order = np.argsort(rng.random((G, n)), axis=1)
    return np.ascontiguousarray(np.take_along_axis(cells, order, axis=1)).view(np.uint64)


def queue_trace(deferred, warps=1):
    """The per-warp queue counts DeferQueue reaches when `warps` warps take the 32-group tiles in turn: (the counts after
    each put, the final drain sizes)."""
    tiles = [int(deferred[i:i + 32].sum()) for i in range(0, len(deferred), 32)]
    peaks, finals = [], []
    for w in range(warps):
        count = 0
        for d in tiles[w::warps]:
            count += d
            peaks.append(count)
            if count >= 32:
                count -= 32
        finals.append(count)
    return peaks, finals


# ----------------------------------------------------------------------------- counts and floors

def counts(vals, rel, ab, infos=None, kinds=None):
    """Path counts of the restated kernel (local route) on rows of n cells."""
    n = vals.shape[1]
    infos = kernel(vals, rel, ab)[2] if infos is None else infos
    c = collections.Counter()
    for inf in infos:
        c["path " + inf["path"]] += 1
        if "extras" in inf:
            c["extras %d,%d" % inf["extras"]] += 1
        if "defer" in inf:
            c["defer: " + inf["defer"]] += 1
        c["uncertified far"] += inf.get("uncertified far", 0)
        c["repair"] += "repair" in inf
        c["middle"] += inf.get("core") == "middle"
        if "tie" in inf:
            c["tie by " + inf["tie"]] += 1
            c["|center| equal"] += "|center| equal" in inf
        for how in inf.get("lent", ()):
            c["lent " + how] += 1
        if n == 64 and inf.get("top start", 0) >= 32:
            c["top start >= 32"] += 1
        if n == 64 and any(s >= 32 for s in inf.get("tie starts", ())) and any(s < 32 for s in inf.get("tie starts", ())):
            c["tie across bit 32"] += 1
        if "quad bits" in inf:
            c["quad %d %s" % (inf["quad bits"][0], "".join("1" if b else "0" for b in inf["quad bits"][1]))] += 1
        if "quad pairs" in inf:
            c["quad pairs by " + inf["quad pairs"]] += 1
        if "pair" in inf:
            c["pair " + inf["pair"]] += 1
    for row in vals:
        xs = sorted(x for x in (u2d(int(u)) for u in row if (int(u) >> 32) not in (NONE_HI, ABSENT_HI)) if math.isfinite(x))
        pairs = [(a, b) for a, b in zip(xs, xs[1:]) if -1.0 < a < 0.0 < b < 1.0]
        c["chain across zero"] += bool(pairs)
        c["chain across zero, close"] += any(_close(a, b, rel, ab) for a, b in pairs)
    return c


def sum_order_residues(vals, rel, ab, infos):
    """Per (z mod 8, (nb, na)): fast-path groups (n = 16, 32) whose cluster of z >= 8 cells, decided with nb extras below v
    and na above, has a numpy mean other than its left-to-right sum (the +0.0 cells of sum_order_row left out)."""
    out = collections.Counter()
    for row, inf in zip(vals, infos):
        if inf.get("path") != "fast":
            continue
        v, m = kernel_group([int(c) for c in row], vals.shape[1], rel, ab)[:2]
        z = (int(m) >> 6) & 0x7F
        xs = sorted(u2d(int(c)) for c in row if (int(c) >> 32) not in (NONE_HI, ABSENT_HI) and int(c) != 0)
        s = -0.0
        for x in xs:
            s += x
        if z >= 8 and len(xs) == z and d2u((0.0 + s) / z) != v:
            out[(z % 8, inf["extras"])] += 1
    return out


def _rows(n, eps_i, per_family=40, seed=0):
    rel, ab = EDGE_EPS[eps_i]
    return family_rows(7000 + 101 * n + 13 * eps_i + seed, n, rel, ab, per_family)


# ----------------------------------------------------------------------------- tests

@pytest.mark.parametrize("n", N_LIST)
def test_brute_force_matches_both_oracles(n):
    """The brute force equals the C oracle bit for bit (value and result word) and the object-level oracle on value and
    confidence, on every family under every EDGE_EPS setting."""
    for i, (rel, ab) in enumerate(EDGE_EPS):
        vals, fam = _rows(n, i, 30)
        ev, em, kinds = brute(vals, rel, ab)
        with np.errstate(all="ignore"):
            ov, om = OC.numeric(vals.view(np.float64), rel, ab)
        check_against(ov, om, ev, em, ("C oracle", n, rel, ab), vals)
        settings = O.OracleSettings(rel_eps=rel, abs_eps=ab)
        for g, row in enumerate(vals):
            live = [u2d(int(c)) for c in row if (int(c) >> 32) not in (NONE_HI, ABSENT_HI)]
            if len(live) < 2:
                continue
            with np.errstate(all="ignore"):
                value, conf = O.numeric(live, settings)
            f = OC.meta_fields(np.array([em[g]]))
            if value is None:
                assert not (int(em[g]) >> 27) & HAS, (n, g)
                continue
            assert d2u(value) == int(ev[g]), (n, rel, ab, g, value, u2d(int(ev[g])))
            assert conf == round(int(f["support"][0]) / len(live), 5), (n, g, conf)


@pytest.mark.parametrize("n", N_LIST)
def test_restated_kernel_equals_brute_force(n):
    """kc_numeric_f64's and kc_numeric_f64_peers' routing restated equals the brute force on every family, under every
    EDGE_EPS setting, and at n = 2 and 4 numeric_pair / numeric_quad and numeric_core agree."""
    for i, (rel, ab) in enumerate(EDGE_EPS):
        vals, fam = _rows(n, i, 30)
        ev, em, _ = brute(vals, rel, ab)
        for route in ("local", "peers"):
            gv, gm, _ = kernel(vals, rel, ab, route)
            check_against(gv, gm, ev, em, ("restated", route, n, rel, ab), vals)


# floors over the four EDGE_EPS settings of one n (family_rows with 40 rows per family)
FLOORS = {
    "extras 1,0": {16: 9, 32: 9}, "extras 0,1": {16: 12, 32: 12}, "extras 2,0": {16: 7, 32: 7},
    "extras 1,1": {16: 10, 32: 10}, "extras 0,2": {16: 7, 32: 7}, "defer: third extra": {16: 10, 32: 10},
    "uncertified far": {16: 7, 32: 7}, "repair": {8: 90, 16: 90, 32: 90, 64: 90},
    "tie by spread": {8: 20, 16: 20, 32: 20, 64: 20}, "|center| equal": {8: 20, 16: 25, 32: 25, 64: 20},
    "lent x10^6": {8: 2, 16: 2, 32: 2, 64: 2}, "lent x10^-6": {8: 1, 16: 1, 32: 1, 64: 1}, "top start >= 32": {64: 7},
    "tie across bit 32": {64: 30}, "middle": {8: 250, 16: 190, 32: 190, 64: 290},
    "defer: no majority": {8: 80, 16: 30, 32: 30}, "defer: shares v's high word": {8: 50, 16: 45, 32: 45},
    "defer: shares a neighbour's high word": {16: 5, 32: 5}, "defer: close neighbour (n = 8)": {8: 60},
    "chain across zero": {n: 13 for n in (2, 4, 8, 16, 32, 64)}, "chain across zero, close": {n: 10 for n in (2, 4, 8, 16, 32, 64)},
    "lent signless": {8: 1, 16: 1, 32: 1, 64: 1},
    **{"lent x10^%d" % k: {8: 1, 16: 1, 32: 1, 64: 1} for k in LENDER_KS},
    **{"pair " + o: {2: 20} for o in ("no value", "single", "no finite", "one finite", "close", "far, larger |hi|", "far, equal |.|",
                                      "far, larger |lo|")},
}


@pytest.mark.parametrize("n", [2, 4, 8, 16, 32, 64])
def test_families_reach_their_paths(n):
    """Host-counted floors: the extras splits, third-extra deferrals and uncertifiable-but-far neighbours at n = 16 and 32;
    repairs, ties decided by spread, equal |centers|, support lent through the signless test and the x 10^k test at every
    k in -6..6 but 0 (the plain test), middle-element majorities, adjacent cells a < 0 < b with |a|, |b| < 1 (close ones
    too); at n = 64 top clusters starting at bit 32 or above and ties across it; at n = 2 every outcome of numeric_pair and
    at n = 4 every close-bit pattern of numeric_quad."""
    total = collections.Counter()
    for i, (rel, ab) in enumerate(EDGE_EPS):
        vals, fam = _rows(n, i)
        total.update(counts(vals, rel, ab))
    print(f"\nn={n}: {dict(sorted(total.items()))}")
    for key, by_n in FLOORS.items():
        if n in by_n:
            assert total[key] >= by_n[n], (key, total[key], by_n[n])
    if n == 4:
        for m in range(1, 5):
            for p in range(2 ** max(m - 1, 0)):
                bits_ = "".join("1" if p >> i & 1 else "0" for i in range(m - 1))
                assert total["quad %d %s" % (m, bits_)] >= 3, (m, bits_, total)
        assert total["quad pairs by order"] >= 5 and total["quad pairs by spread"] >= 5, total


SPLITS = [(0, 0), (1, 0), (0, 1), (2, 0), (1, 1), (0, 2)]


@pytest.mark.parametrize("n", [16, 32])
def test_summation_order_rows(n):
    """Family 4 in full (the rows tests/test_gpu_numeric_edges.py runs through the fast kernels): under the two settings
    where extras can be close to v, every (z mod 8, nb, na) with z >= 8 is decided on the fast path with those extras by a
    cluster whose numpy mean differs from a left-to-right sum, at least once per setting at n = 32.  At n = 16 a cluster of
    z = 9 with two extras holds 7 copies of v, fewer than the 8 cells the "at least half" guess needs, so residue 1 is
    reached with one extra or none only."""
    total = collections.Counter()
    for i in (0, 2):
        rel, ab = EDGE_EPS[i]
        rows, cases = sum_order_rows(n, i)
        gv, gm, infos = kernel(rows, rel, ab)
        ev, em, _ = brute(rows, rel, ab)
        check_against(gv, gm, ev, em, ("sum order", n, rel, ab), rows)
        total.update(sum_order_residues(rows, rel, ab, infos))
    print(f"\nn={n}: fast-path clusters per (z mod 8, extras) that differ from a left-to-right sum: {dict(sorted(total.items()))}")
    for t in range(8):
        for split in SPLITS:
            if n == 16 and t == 1 and sum(split) == 2:
                continue
            assert total[(t, split)] >= n // 16, (t, split, dict(total))


@pytest.mark.parametrize("n", [8, 16, 32])
def test_queue_layouts(n):
    """Family 8: every tile defers exactly the groups its layout says, and one warp's queue reaches exactly 32, 33 to 63
    (the overflow re-read) and final drains of 1 and 31."""
    rel, ab = EDGE_EPS[0]
    peaks, finals = collections.Counter(), collections.Counter()
    for name, lay in QUEUE_LAYOUTS.items():
        for G in (32 * 5 + 1, 32 * 5 + 31):
            vals = queue_rows(n, G, lay, G + n)
            gv, gm, infos = kernel(vals, rel, ab)
            ev, em, _ = brute(vals, rel, ab)
            check_against(gv, gm, ev, em, ("queue", n, name, G), vals)
            deferred = np.array([inf["path"] == "deferred" for inf in infos])
            for t in range(-(-G // 32)):
                want = min(lay[t % len(lay)], G - 32 * t)
                got = int(deferred[32 * t:32 * t + 32].sum())
                assert got == want or (32 * t + 32 > G and got <= want), (name, G, t, got, want)
            for warps in (1, 2):
                p, f = queue_trace(deferred, warps)
                peaks.update(p)
                finals.update(f)
            vs = gv.view(np.float64)
            assert len(set(vs.tolist())) == G, "values are not distinct"
    print(f"\nn={n}: queue counts {dict(sorted(peaks.items()))}; final drains {dict(sorted(finals.items()))}")
    assert peaks[32] >= 3 and sum(peaks[k] for k in range(33, 64)) >= 3 and finals[1] >= 1 and finals[31] >= 1


def _mutation_rows(n, i):
    """The rows the mutation search runs at n under EDGE_EPS[i]: the families, and at n = 16 and 32 family 4 in full."""
    vals, _ = _rows(n, i)
    if n in (16, 32) and i in (0, 2):
        vals = np.concatenate([vals, sum_order_rows(n, i)[0]])
    return vals


def test_mutated_kernel_goes_wrong_on_the_families():
    """Each MUTATION of the restated kernel gives a wrong value or result word on some family group, and the unmutated
    restatement gives none on the same rows (both routes).  UNCATCHABLE lists the edits that cannot change an output, with
    the reason beside it."""
    where = {"decide": (8, 16, 32), "certainly_far": (8, 16, 32), "walk": (16, 32), "finish": (16, 32), "far_bit": (8, 16, 64, 5),
             "core": (64, 16, 32, 5, 8), "tie": (8, 16, 64, 32), "is_close_pow10": (16, 32, 64), "np_mean16": (16, 9, 15),
             "pair": (2,), "quad": (4,)}
    data = {}
    wrong = collections.Counter()

    def mismatches(key, mut, route):
        vals, (ev, em, _) = data[key]
        gv, gm, _ = kernel(vals, *EDGE_EPS[key[1]], route, mut)
        no_value = ((em >> 27) & HAS) == 0
        return int((~((gm == em) & ((gv == ev) | (no_value & nan_bits(gv) & nan_bits(ev))))).sum())

    for mut in MUTATIONS:
        found = 0
        for n in where[mut.split(":")[0]]:
            for i in range(len(EDGE_EPS)):
                if (n, i) not in data:
                    vals = _mutation_rows(n, i)
                    data[n, i] = (vals, brute(vals, *EDGE_EPS[i]))
                    for route in ("local", "peers"):
                        wrong[None] += mismatches((n, i), None, route)
                for route in ("local", "peers") if mut.startswith(("core", "tie", "is_close", "np_mean16", "far_bit")) else ("local",):
                    found += mismatches((n, i), mut, route)
                if found >= 3 and mut not in UNCATCHABLE:
                    break
            if found >= 3 and mut not in UNCATCHABLE:
                break
        wrong[mut] = found
    print("\ngroups each mutation gets wrong (search stops at 3):", dict(wrong))
    assert wrong[None] == 0, wrong[None]
    for mut in MUTATIONS:
        if mut not in UNCATCHABLE:
            assert wrong[mut] >= 1, (mut, dict(wrong))
