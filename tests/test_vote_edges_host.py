"""CPU: K1's vote (kc_vote.cuh) at its decision edges, without a GPU.

vote_core decides most groups with shortcuts whose boundaries decide the answer: a bitwise-majority guess over 1, 3, 8 (cell 0
counted twice), 15 or 27 chosen cells; the strict-majority test 2 * cnt > voters that accepts the guess, with ffs of the
equality mask as its first-seen index (64-bit at n = 64); and the first-seen scan that stops once the unvisited cells are
fewer than the best count, so that a class of equal size visited last still sets TIE.  This file holds the edge families the
GPU tests (tests/test_gpu_vote_edges.py) run through every K1 kernel, a vectorised brute force (every class counted, no
guess, no early stop), and a numpy restatement of vote_core's routing that reports which path each group takes.  It checks
the brute force against the C oracle and a plain Counter loop, that each family reaches the path it is built for, and that
the restatement goes wrong on the families when one of its decisions is mutated.

A family row is n raw cells for one group (code >= 0, None -1, absent -2) built for that group's none_code nc (>= 0: None
votes as nc).  `wide` rows use int32 codes up to 2^31 - 1; the others fit int8 cells (codes <= 127)."""
import collections
import random

import numpy as np
import pytest

from oracle import columnar as OC
from tests.test_weighted_edges_host import map_cells, pack_meta

N_LIST = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64]
FAMILIES = (1, 2, 3, 4, 5, 6)
LANES = (0, 31, 32, 63)  # the lanes on both sides of the 64-bit masks' halves
I32_MAX = 2 ** 31 - 1


def pow2(n):
    p = 1
    while p < n:
        p *= 2
    return p


# ----------------------------------------------------------------------------- the brute force and a Counter loop

def brute(codes, nc=None):
    """voting_consensus of every group by counting all its classes: codes int [G, n] raw cells, nc int [G] (None: no
    none_code).  Returns dict(win, meta) and the voting codes x."""
    codes = np.asarray(codes, dtype=np.int32)
    G, n = codes.shape
    nc = np.full(G, -1, np.int32) if nc is None else np.asarray(nc, dtype=np.int32)
    x = map_cells(codes, nc)
    vote = x >= 0
    cnt = np.zeros((G, n), np.int64)
    later = np.zeros((G, n), bool)  # cell i has an earlier voting cell of its class
    ar = np.arange(n)
    for j in range(n):
        m = vote & vote[:, j:j + 1] & (x == x[:, j:j + 1])
        cnt += m
        later |= m & (ar > j)
    first = vote & ~later
    cf = np.where(first, cnt, 0)
    best = cf.max(axis=1)
    at_best = first & (cf == best[:, None])
    idx = np.argmax(at_best, axis=1)  # the first-seen class among the largest
    tie = at_best.sum(axis=1) > 1
    voters = vote.sum(axis=1)
    present = (codes >= -1).sum(axis=1)
    has = voters > 0
    rows = np.arange(G)
    win = np.where(has, x[rows, idx], -1).astype(np.int32)
    meta = pack_meta(np.where(has, idx, 0), np.where(has, best, 0), voters, present,
                     np.where(has, 1 | np.where(tie, 4, 0), 0))
    return dict(win=win, meta=meta, x=x)


def counter_vote(row, nc):
    """One group the plain way: the voting values in cell order into a Counter, most_common(1) (the first inserted among
    the largest), TIE when another class has as many votes."""
    present = sum(1 for v in row if v >= -1)
    votes = [(i, nc if v == -1 else v) for i, v in enumerate(row) if v >= 0 or (v == -1 and nc >= 0)]
    if not votes:
        return -1, int(pack_meta(np.int64(0), 0, 0, present, 0))
    counts = collections.Counter(v for _, v in votes)
    code, k = counts.most_common(1)[0]
    tie = sum(1 for c in counts.values() if c == k) > 1
    first = next(i for i, v in votes if v == code)
    return code, int(pack_meta(np.int64(first), k, len(votes), present, 1 | (4 if tie else 0)))


# ----------------------------------------------------------------------------- vote_core restated

def _maj(a, b, c):
    return (a & b) | (a & c) | (b & c)


def guess(x, NP):
    """guess_mode<NP>: the bitwise majority tree over the cells it reads, on uint32 bit patterns."""
    u = np.asarray(x, dtype=np.int32).view(np.uint32)
    c = lambda i: u[:, i]  # noqa: E731
    if NP >= 27:
        t = [_maj(c(3 * i), c(3 * i + 1), c(3 * i + 2)) for i in range(9)]
        r = _maj(_maj(t[0], t[1], t[2]), _maj(t[3], t[4], t[5]), _maj(t[6], t[7], t[8]))
    elif NP >= 15:
        a, b, cc, d, e = (_maj(c(3 * i), c(3 * i + 1), c(3 * i + 2)) for i in range(5))
        s, cy = a ^ b ^ cc, _maj(a, b, cc)
        r = (cy & (s | d | e)) | (s & d & e)
    elif NP >= 8:
        r = _maj(_maj(c(0), c(1), c(2)), _maj(c(3), c(4), c(5)), _maj(c(6), c(7), c(0)))
    elif NP >= 3:
        r = _maj(c(0), c(1), c(2))
    else:
        r = c(0)
    return np.ascontiguousarray(r, dtype=np.uint32).view(np.int32)


def guess_cells(NP):
    """The cells guess_mode<NP> reads."""
    return list(range(27 if NP >= 27 else 15 if NP >= 15 else 8 if NP >= 8 else 3 if NP >= 3 else 1))


MUTATIONS = ("stop <=", "majority >=", "TIE kept on a larger class", "32-bit ffs at n = 64")


def pad(codes, NP):
    codes = np.asarray(codes, dtype=np.int32)
    G, n = codes.shape
    return codes if n == NP else np.concatenate([codes, np.full((G, NP - n), -2, np.int32)], axis=1)


def core(codes, nc, NP, mutation=None):
    """vote_core<NP, HAS_NC> on rows padded to NP cells (absent beyond n), optionally with one of MUTATIONS.  Returns the
    results and the routing: path[g] = 'absent' (some cell absent: scan), 'guess' (decided by the majority test), or the
    reason the scan runs: 'negative' (the guess is negative), 'not present', 'minority' (a present minority), 'half'
    (exactly half of the voters); boundary[g]: the scan finished a class with as many unvisited voting cells left as its
    best count (where it has to go on)."""
    raw = pad(codes, NP)
    G = raw.shape[0]
    nc = np.full(G, -1, np.int32) if nc is None else np.asarray(nc, dtype=np.int32)
    x = map_cells(raw, nc)
    absent = (raw < -1).any(axis=1)
    voters = (x >= 0).sum(axis=1)
    c = guess(x, NP)
    eq = x == c[:, None]
    cnt = eq.sum(axis=1)
    maj = 2 * cnt >= voters if mutation == "majority >=" else 2 * cnt > voters
    fast = ~absent & (c >= 0) & maj
    fidx = np.argmax(eq, axis=1)
    if mutation == "32-bit ffs at n = 64" and NP == 64:  # __ffs((int)m): 0 for a mask without a low bit, index -1 & 0x3F
        low = eq[:, :32]
        fidx = np.where(low.any(axis=1), np.argmax(low, axis=1), 63)
    present = np.where(absent, (raw >= -1).sum(axis=1), NP)
    swin, smeta, boundary = scan(x, present, mutation)
    win = np.where(fast, c, swin).astype(np.int32)
    meta = np.where(fast, pack_meta(fidx, cnt, voters, NP, 1), smeta).astype(np.uint32)
    path = np.where(absent, "absent", np.where(fast, "guess", np.where(
        c < 0, "negative", np.where(cnt == 0, "not present", np.where(2 * cnt == voters, "half", "minority")))))
    return dict(win=win, meta=meta, path=path, boundary=boundary & ~fast)


def scan(x, present, mutation=None):
    """vote_scan: classes in first-seen order, a later class must be strictly larger, stop once fewer unvisited voting
    cells remain than the best count."""
    G, N = x.shape
    ar = np.arange(N)
    live = x >= 0
    voters = live.sum(axis=1)
    best_cnt = np.zeros(G, np.int64)
    best_idx = np.zeros(G, np.int64)
    best_code = np.full(G, -1, np.int64)
    tie = np.zeros(G, bool)
    boundary = np.zeros(G, bool)
    for i in range(N):
        act = live[:, i].copy()
        if not act.any():
            continue
        eq = act[:, None] & (x == x[:, i:i + 1]) & (ar >= i)
        k = eq.sum(axis=1)
        gt = act & (k > best_cnt)
        same = act & (k == best_cnt)
        best_idx = np.where(gt, i, best_idx)
        best_code = np.where(gt, x[:, i], best_code)
        best_cnt = np.where(gt, k, best_cnt)
        tie = np.where(gt, tie if mutation == "TIE kept on a larger class" else False, tie | same)
        live &= ~eq
        rem = live.sum(axis=1)
        boundary |= act & (rem > 0) & (rem == best_cnt)
        stop = act & ((rem <= best_cnt) if mutation == "stop <=" else (rem < best_cnt))
        live &= ~stop[:, None]
    has = best_cnt > 0
    meta = pack_meta(best_idx, best_cnt, voters, present, np.where(has, 1 | np.where(tie, 4, 0), 0))
    return np.where(has, best_code, -1), meta, boundary


# ----------------------------------------------------------------------------- the edge families

def _codes(r, k, wide, avoid=()):
    """k distinct codes: small ones, and with `wide` also large int32 ones."""
    out = []
    while len(out) < k:
        if wide and r.random() < 0.6:
            c = r.choice([r.randrange(1000, I32_MAX), (1 << r.randrange(10, 31)) - r.randrange(0, 2), I32_MAX, 1 << 30])
        else:
            c = r.randrange(0, 128)
        if c not in out and c not in avoid:
            out.append(c)
    return out


class Row:
    """n cells being filled: put() places a class, fill() the rest."""

    def __init__(self, r, n, nc):
        self.r, self.n, self.nc, self.cells = r, n, nc, [None] * n

    def free(self, lo=0, hi=None):
        return [i for i in range(lo, self.n if hi is None else hi) if self.cells[i] is None]

    def put(self, code, count, first=None, lo=0):
        """count cells of `code`, the first at `first` (if given) and the rest after it, else anywhere from lo."""
        if first is not None:
            self.cells[first] = code
            rest = self.r.sample(self.free(first + 1), count - 1)
        else:
            rest = self.r.sample(self.free(lo), count)
        for i in rest:
            self.cells[i] = code

    def spell_none(self, code, k):
        """Spell k cells of `code` as None: they still vote as it through nc == code."""
        if self.nc == code:
            idx = [i for i, v in enumerate(self.cells) if v == code]
            for i in self.r.sample(idx, min(k, len(idx))):
                self.cells[i] = -1

    def fill(self, cap, used, wide):
        """The free cells: non-voting None (when nc < 0), or classes of at most `cap` cells with new codes; absent only where
        neither fits."""
        free = self.free()
        self.r.shuffle(free)
        while free:
            if self.nc < 0 and (cap < 1 or self.r.random() < 0.35):
                self.cells[free.pop()] = -1
                continue
            if cap < 1:
                self.cells[free.pop()] = -2
                continue
            code = _codes(self.r, 1, wide, avoid=set(used) | {self.nc})[0]
            used.append(code)
            for _ in range(min(len(free), self.r.randint(1, cap))):
                self.cells[free.pop()] = code

    def done(self):
        assert None not in self.cells
        return self.cells


def _lane(r, n):
    opts = [p for p in LANES if p < n]
    return r.choice(opts) if opts and r.random() < 0.6 else r.randrange(n)


def fam_ties(r, n, nc, wide):
    """Family 1: k >= 2 classes of exactly s cells each in a random first-seen order, one of them starting at lane 0, 31, 32
    or 63 (n = 64) or anywhere; the rest smaller classes or non-voters.  With nc >= 0 one tied class is often nc, spelled
    None in some of its cells (the tie exists only through nc)."""
    if n < 2:
        return fam_mixed(r, n, nc, wide)
    lane = _lane(r, n)
    k = r.choice([2, 2, 3, 4])
    s = max(1, min(n // k, n - lane, r.choice([1, 2, 3, max(1, n // k)])))
    k = min(k, n // s)
    row = Row(r, n, nc)
    codes = _codes(r, k, wide, avoid={nc})
    if nc >= 0 and r.random() < 0.6:
        codes[r.randrange(k)] = nc
    t = r.randrange(k)
    row.put(codes[t], s, first=lane)
    for j in range(k):
        if j != t:
            row.put(codes[j], s)
    for code in codes:
        row.spell_none(code, r.randint(1, s))
    row.fill(s - 1, codes, wide)
    return row.done()


def fam_majority(r, n, nc, wide):
    """Family 2: the class the guess reads most holds exactly half of the voters, half + 1, or (odd voters) the smallest
    strict majority; the others are one class (a tie at half) or several.  None cells do not vote, vote as that class, or
    vote as the other one."""
    if n < 2:
        return fam_mixed(r, n, nc, wide)
    row = Row(r, n, nc)
    nones = r.randint(0, n - 2) if nc < 0 and r.random() < 0.5 else 0
    v = n - nones
    g = {0: v // 2, 1: v // 2 + 1, 2: (v + 1) // 2}[r.randrange(3)]
    g = max(1, min(g, v))
    main, other = _codes(r, 2, wide, avoid={nc})
    if nc >= 0:
        pick = r.random()
        main, other = (nc, other) if pick < 0.4 else (main, nc) if pick < 0.7 else (main, other)
    sampled = [i for i in guess_cells(pow2(n)) if i < n]
    r.shuffle(sampled)
    for i in sampled[:g]:
        row.cells[i] = main
    if g > len(sampled):
        row.put(main, g - len(sampled))
    for i in r.sample(row.free(), nones):
        row.cells[i] = -1
    if r.random() < 0.5:
        row.put(other, v - g)
    else:
        row.fill(max(1, min(v - g, g) - 1), [main, other], wide)
    row.spell_none(main, r.randint(0, g))
    row.spell_none(other, r.randint(0, n))
    return row.done()


def _fooling(r, wide):
    """p, q, r with a bitwise majority z that is none of them: z with three disjoint bit masks flipped."""
    bits = list(range(31 if wide else 7))
    while True:
        z = r.randrange(0, 1 << len(bits))
        r.shuffle(bits)
        cut = sorted(r.sample(range(1, len(bits)), 2))
        groups = [bits[:cut[0]], bits[cut[0]:cut[1]], bits[cut[1]:]]
        masks = [sum(1 << b for b in r.sample(g, r.randint(1, min(3, len(g))))) for g in groups]
        pqr = [z ^ m for m in masks]
        if all(0 <= c <= (I32_MAX if wide else 127) for c in pqr):
            return z, pqr


def fam_fooled(r, n, nc, wide):
    """Family 3: the guess is fooled.  The cells it reads hold p, q, r whose bitwise majority is a code z that is (a) absent
    from the group, (b) a present minority, or the cells read are mostly None so that the guess is negative (c, nc < 0).
    The true mode T fills the triples the guess's tree outvotes and the cells it never reads.  At n = 8 the triple
    (6, 7, 0) reads cell 0 a second time."""
    NP = pow2(n)
    if NP < 4:
        return fam_mixed(r, n, nc, wide)
    z, pqr = _fooling(r, wide)
    if n == 64 and nc < 0 and r.random() < 0.3:  # (d) the guess is right, from codes that are not its
        return _fooled_high(r, z, pqr)
    variant = r.choice("abc") if nc < 0 else r.choice("ab")
    T = _codes(r, 1, wide, avoid=set(pqr) | {z, nc})[0]
    if nc >= 0 and r.random() < 0.5 and nc not in pqr and nc != z:
        T = nc
    trip = lambda: r.sample(pqr, 3) if variant != "c" else [-1, -1, r.choice(pqr + [T])]  # noqa: E731
    cells = [T] * NP  # built at NP, cut to n (rows of other n are padded absent: the scan)
    if NP >= 27:  # 9 triples in 3 groups: two triples in each of two groups give z
        for grp in r.sample(range(3), 2):
            for t in r.sample(range(3), 2):
                cells[9 * grp + 3 * t:9 * grp + 3 * t + 3] = trip()
    elif NP >= 15:  # 3 of the 5 triples under maj5
        for t in r.sample(range(5), 3):
            cells[3 * t:3 * t + 3] = trip()
    elif NP >= 8:  # triples (0, 1, 2) and (6, 7, 0): cell 0 counts twice
        a = trip()
        cells[0:3] = a
        b = [v for v in (pqr if variant != "c" else [-1, -1]) if v != a[0]] if variant != "c" else [-1, a[2]]
        cells[6], cells[7] = b[0], b[1]
    else:
        cells[0:3] = trip()
    cells = cells[:n]
    if variant == "b":
        spots = [i for i in range(n) if cells[i] == T] or list(range(n))
        for i in r.sample(spots, min(len(spots), r.randint(1, 2))):
            cells[i] = z
    if T == nc:
        for i in [i for i in range(n) if cells[i] == T][:r.randint(0, 3)]:
            cells[i] = -1
    return cells


def _fooled_high(r, T, pqr):
    """n = 64: T fills most of cells 32-63 and holds a strict majority, the guess's 27 cells hold p, q, r (whose bitwise
    majority is T) or None: the guess finds T although none of its cells holds it, and the majority test decides a winner
    whose first cell is in the high half of the 64-bit mask."""
    cells = [-1] * 64
    for grp in r.sample(range(3), 2):
        for t in r.sample(range(3), 2):
            cells[9 * grp + 3 * t:9 * grp + 3 * t + 3] = r.sample(pqr, 3)
    first = r.randint(32, 40)
    for i in range(first, 64):
        cells[i] = T if (i == first or r.random() < 0.9) else r.choice(pqr + [-1])
    return cells


def fam_stop(r, n, nc, wide):
    """Family 4: the scan's stop.  Class A (s cells) is seen first, then classes of at most s cells (sometimes one of s: an
    early tie), then B, whose first cell comes after every other class's first cell, with s cells (it must set TIE: the scan
    reaches it with exactly s cells left), s - 1 (no TIE) or s + 1 (B wins from a late first cell, at n = 64 often 33 or
    more)."""
    if n < 3:
        return fam_ties(r, n, nc, wide)
    d = r.choice([0, 0, -1, 1])
    lo = 33 if n == 64 and r.random() < 0.6 else 1
    b0 = r.randint(min(lo, n - 2), n - 2)
    s = r.randint(1, max(1, min(b0, n - b0 - max(d, 0), 12)))
    nb = s + d
    if nb < 1:
        s, nb = 2, 1
    A, B = _codes(r, 2, wide, avoid={nc})
    if nc >= 0 and r.random() < 0.5:
        A, B = (nc, B) if r.random() < 0.5 else (A, nc)
    row = Row(r, n, nc)
    row.cells[b0] = B
    for i in r.sample(row.free(b0 + 1), min(nb - 1, len(row.free(b0 + 1)))):
        row.cells[i] = B
    first_a = r.choice(row.free(0, b0))
    row.cells[first_a] = A
    for i in r.sample(row.free(first_a + 1), min(s - 1, len(row.free(first_a + 1)))):
        row.cells[i] = A
    # the others: classes started before b0, of at most s - 1 cells (one of s at times), or non-voters
    cap, used, open_ = s - 1, [A, B], []
    for i in row.free():
        if i < b0 and (not open_ or r.random() < 0.4):
            size = s if (r.random() < 0.15 and cap >= 0) else cap
            if size >= 1:
                code = _codes(r, 1, wide, avoid=set(used) | {nc})[0]
                used.append(code)
                open_.append([code, size])
        live = [o for o in open_ if o[1] > 0]
        if live and (nc >= 0 or r.random() < 0.8):
            o = r.choice(live)
            row.cells[i] = o[0]
            o[1] -= 1
        else:
            row.cells[i] = -1 if nc < 0 else -2
    row.spell_none(A, r.randint(0, s))
    row.spell_none(B, r.randint(0, nb))
    return row.done()


def fam_range(r, n, nc, wide):
    """Family 5: codes at the ends of the range (0, 1, 2^k - 1, 2^k, 2^30, 2^31 - 1; 63 and 127 in int8 cells), nc often one
    of the row's codes, with None cells."""
    pal = [0, 1, 2, 3, 7, 8, 15, 16, 31, 32, 63, 64, 127]
    if wide:
        k = r.randrange(1, 31)
        pal = [0, 1, (1 << k) - 1, 1 << k, 1 << 30, I32_MAX, (1 << 30) - 1, (1 << 30) + 1, 1 << 16]
    k = min(n, r.choice([1, 2, 3, 4]))
    codes = r.sample(pal, k)
    if nc >= 0 and r.random() < 0.5 and nc not in codes:
        codes[r.randrange(k)] = nc
    cells = [r.choice(codes) for _ in range(n)]
    for i in range(n):
        if r.random() < 0.15:
            cells[i] = -1
    if nc >= 0:  # a None votes as nc: keep nc's cells spelled both ways
        cells = [(-1 if (v == nc and r.random() < 0.5) else v) for v in cells]
    return cells


def fam_mixed(r, n, nc, wide):
    """Family 6: None and absent cells: one absent cell at lane 0, 31, 32 or 63 (a strict majority sent to the absent path
    with it), every cell absent, every cell None, a single voter, present cells without a voter."""
    v = r.randrange(6)
    A, B = _codes(r, 2, wide, avoid={nc})
    if v == 0:  # a strict majority, one absent cell
        cells = [A if r.random() < 0.75 else B for _ in range(n)]
        cells[_lane(r, n)] = -2
        return cells
    if v == 1:
        return [-2] * n
    if v == 2:
        return [-1] * n
    if v == 3:  # one voter among None / absent cells
        cells = [-1 if (nc < 0 and r.random() < 0.5) else -2 for _ in range(n)]
        cells[_lane(r, n)] = r.choice([A, -1]) if nc >= 0 else A
        return cells
    if v == 4:  # None and absent only
        cells = [r.choice([-1, -2]) for _ in range(n)]
        cells[r.randrange(n)] = -1
        return cells
    cells = [r.choice([A, A, B, -1]) for _ in range(n)]  # absent at several of the lanes
    for p in LANES:
        if p < n and r.random() < 0.7:
            cells[p] = -2
    return cells


MAKERS = {1: fam_ties, 2: fam_majority, 3: fam_fooled, 4: fam_stop, 5: fam_range, 6: fam_mixed}


def nc_table(r, F, wide):
    """A none_code entry per field: -1 interleaved with 0, small codes, 127 / 2^31 - 1 and random codes."""
    big = I32_MAX if wide else 127
    opts = [-1, 0, 1, big, -1, r.randrange(0, 128), 63, -1, r.randrange(0, big + 1)]
    return np.array([opts[(f + r.randrange(2)) % len(opts)] if f else -1 for f in range(F)], dtype=np.int32) \
        if F > 1 else np.array([r.choice([0, big, 5])], dtype=np.int32)


def family_rows(seed, n, per_family, table=None, wide=True, families=FAMILIES):
    """per_family rows of each family, family after family: codes int32 [G, n], family [G], nc [G] (table[g % F], or -1
    without a table).  Each row is built for its own group's nc."""
    r = random.Random(seed)
    G = per_family * len(families)
    F = len(table) if table is not None else 1
    ncg = np.array([int(table[g % F]) for g in range(G)] if table is not None else [-1] * G, dtype=np.int32)
    fam = np.repeat(np.array(families), per_family)
    codes = np.array([MAKERS[f](r, n, int(ncg[g]), wide) for g, f in enumerate(fam)], dtype=np.int32).reshape(G, n)
    assert codes.min() >= -2 and (wide or codes.max() <= 127)
    return codes, fam, ncg


def counts(codes, ncg, ref=None):
    """The floors' counts on the host for rows of n cells: vote_core's routing at NP = the next power of two (cells beyond n
    absent, as the direct kernels pad them), and the brute force's flags."""
    n = codes.shape[1]
    ref = brute(codes, ncg) if ref is None else ref
    rt = core(codes, ncg, pow2(n))
    fast_scan = rt["path"] != "absent"
    fast_scan &= rt["path"] != "guess"
    return {"scan, no absent cell": int(fast_scan.sum()),
            "TIE": int(((ref["meta"] >> 29) & 1).sum()),
            "TIE, no absent cell": int((((ref["meta"] >> 29) & 1) == 1)[rt["path"] != "absent"].sum()),
            "scan at remaining == best": int(rt["boundary"].sum()),
            "... no absent cell": int((rt["boundary"] & (rt["path"] != "absent")).sum()),
            "first index >= 32": int((((ref["meta"] & 0x3F) >= 32) & (ref["win"] >= 0)).sum())}


def check_against(got_win, got_meta, ref, what=""):
    bad = np.flatnonzero((np.asarray(got_win).astype(np.int64) != ref["win"])
                         | (np.asarray(got_meta).astype(np.int64) != ref["meta"].astype(np.int64)))
    assert not bad.size, (what, bad.size, bad[:8], OC.meta_fields(np.asarray(got_meta)[bad[:3]].astype(np.uint32)),
                          OC.meta_fields(ref["meta"][bad[:3]]))


# ----------------------------------------------------------------------------- tests

def _cases(n, per_family, seed):
    """Each family without a table and with tables of 3 and 7 fields, int32-wide and int8-narrow codes."""
    for wide in (True, False):
        for F in (None, 3, 7):
            r = random.Random(seed + 17 * (F or 0) + wide)
            table = nc_table(r, F, wide) if F else None
            yield (wide, F), family_rows(seed + 101 * (F or 0) + wide, n, per_family, table, wide)


@pytest.mark.parametrize("n", N_LIST)
def test_brute_force_matches_c_oracle_and_counter(n):
    for what, (codes, fam, ncg) in _cases(n, 60, 1000 + n):
        ref = brute(codes, ncg)
        win, meta = OC.vote(codes, ncg[:what[1]] if what[1] else None)
        check_against(win, meta, ref, ("C oracle", n) + what)
        for g in range(0, len(codes), 5):
            assert counter_vote([int(v) for v in codes[g]], int(ncg[g])) == (ref["win"][g], ref["meta"][g]), (n, what, g)


@pytest.mark.parametrize("NP", [1, 2, 4, 8, 16, 32, 64])
def test_guess_cells_and_restated_core_equal_brute_force(NP):
    """The restated vote_core (guess, majority test, scan) equals the brute force on every family at NP, and the guess reads
    only the cells guess_cells lists."""
    rng = np.random.default_rng(NP)
    for what, (codes, fam, ncg) in _cases(NP, 80, 2000 + NP):
        got = core(codes, ncg, NP)
        check_against(got["win"], got["meta"], brute(codes, ncg), ("core", NP) + what)
    x = rng.integers(0, 1 << 20, (500, NP)).astype(np.int32)
    y = x.copy()
    rest = [i for i in range(NP) if i not in guess_cells(NP)]
    y[:, rest] = rng.integers(0, 1 << 20, (500, len(rest)))
    assert np.array_equal(guess(x, NP), guess(y, NP))


# minimum number of groups of each family that reach a path, over _cases(NP, 80) (12 x 80 rows per family)
REACH = {1: [("scan", "any", 200)],
         2: [("half", 4, 60), ("guess", 2, 60), ("minority", 8, 10)],
         3: [("not present", 4, 100), ("minority", 4, 60), ("negative", 4, 30)],
         4: [("boundary", 4, 120)],
         5: [("scan", "any", 100)],
         6: [("absent", "any", 300)]}


@pytest.mark.parametrize("NP", [2, 4, 8, 16, 32, 64])
def test_families_reach_their_paths(NP):
    """Each family sends its groups where it is built to: ties and stops into the scan (past a remaining == best boundary),
    the majority family onto both sides of 2 * cnt > voters, the fooled family past guesses that are absent, a minority or
    negative, the mixtures onto the absent path."""
    got = collections.defaultdict(collections.Counter)
    for _, (codes, fam, ncg) in _cases(NP, 80, 3000 + NP):
        rt = core(codes, ncg, NP)
        for f in FAMILIES:
            m = fam == f
            got[f].update(rt["path"][m].tolist())
            got[f]["boundary"] += int(rt["boundary"][m].sum())
            got[f]["scan"] += int((~np.isin(rt["path"][m], ["guess", "absent"])).sum())
    print(f"\nNP={NP}: " + "; ".join(f"family {f}: {dict(got[f])}" for f in FAMILIES))
    for f, floors in REACH.items():
        for key, min_np, floor in floors:
            if min_np == "any" or NP >= min_np:
                assert got[f][key] >= floor, (f, key, dict(got[f]))


def test_mutated_core_goes_wrong_on_the_families():
    """The families catch each mutation of the restated vote_core: the scan stopping at remaining == best (a late class of
    equal size loses its TIE), the majority test accepting exactly half, TIE surviving a strictly larger class, and a 32-bit
    ffs of the equality mask at n = 64.  The unmutated restatement agrees everywhere."""
    wrong = collections.Counter()
    for NP in (8, 16, 32, 64):
        for _, (codes, fam, ncg) in _cases(NP, 80, 4000 + NP):
            ref = brute(codes, ncg)
            for mutation in (None,) + MUTATIONS:
                got = core(codes, ncg, NP, mutation)
                wrong[mutation] += int(((got["win"] != ref["win"]) | (got["meta"] != ref["meta"])).sum())
    print("\ngroups each mutation gets wrong:", dict(wrong))
    assert wrong[None] == 0, wrong
    for mutation in MUTATIONS:
        assert wrong[mutation] >= 20, (mutation, dict(wrong))


def test_counts_at_n32_and_n64():
    """Without absent cells the families hold hundreds of TIE groups and of scans that reach remaining == best at a class
    boundary, and at n = 64 winners whose first cell is in the high half of the mask."""
    for n in (32, 64):
        codes, fam, ncg = family_rows(5000 + n, n, 300)
        c = counts(codes, ncg)
        print(f"\nn={n}: {c}")
        assert c["TIE, no absent cell"] >= 200 and c["... no absent cell"] >= 200, c
        if n == 64:
            assert c["first index >= 32"] >= 50, c
