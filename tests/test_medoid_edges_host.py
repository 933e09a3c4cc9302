"""CPU: K4's Levenshtein medoid (kc_medoid.cuh, medoid_kernel) at its decision edges, without a GPU.

medoid_kernel decides a group of normalised strings through choices whose edges random phrases reach only by chance: string
classes from a (FNV-1a hash, length) match for k <= 32, confirmed character by character, with an exact scan as the fall-back
and for k > 32; Myers' bit-parallel distance with the shorter string as the pattern, a 32-bit word up to 32 characters and a
64-bit one above, d = tl for an empty pattern; the similarity 1 - d / tl floored at 1e-8; row sums in numpy's pairwise order
with the diagonal as +0.0; the first maximum within a lane (rows i and i + 32 share one) and the lowest index across lanes.

This file holds the edge families the GPU tests (tests/test_gpu_medoid_edges.py) run through K4, the JSON paths and the
alignment pre-pass; a brute force (a numpy Levenshtein DP, the k x k matrix with a NaN diagonal, np.nanmean, np.argmax); and a
restatement of medoid_kernel.  It checks the brute force against the Python and native edit distances and the C oracle, the
restatement against the brute force, that the restatement goes wrong on the families under each of eight mutations, and
host-counted floors, so that a generator change cannot quietly make the cases easy.  All strings are normalised ([a-z0-9])."""
import collections
import ctypes
import json
import random

import numpy as np

from oracle import columnar as OC
from oracle.consensus_py import edit_distance
from tests.alignsim_cases import assert_matrices
from tests.helpers import _fnv1a, _fnv_collision

ALNUM = "abcdefghijklmnopqrstuvwxyz0123456789"
PATTERN_LENGTHS = (1, 31, 32, 33, 63, 64)
FLOOR = 1e-8
FAMILIES = ("word", "choice", "empty", "classes", "ties", "order")

# ----------------------------------------------------------------------------- the brute force


def _batches(pairs):
    """Pairs (pattern, text) with len(pattern) <= len(text) in batches of patterns and texts of similar lengths."""
    by = collections.defaultdict(list)
    for p, t in pairs:
        by[len(p).bit_length(), len(t).bit_length()].append((p, t))
    for _, items in sorted(by.items()):
        for s in range(0, len(items), 4096):
            yield items[s:s + 4096]


def _codes(strings, width, pad):
    """[a-z0-9] -> 0..35 in a [len, width] array, `pad` beyond each string's end."""
    out = np.full((len(strings), max(width, 1)), pad, np.int16)
    for r, s in enumerate(strings):
        if s:
            b = np.frombuffer(s.encode(), np.uint8).astype(np.int16)
            out[r, :len(s)] = np.where(b >= ord("a"), b - ord("a"), b - ord("0") + 26)
    return out


def dp_distances(pairs):
    """Levenshtein distances of (pattern, text) pairs by the textbook DP, one text row at a time for the whole batch; the
    within-row recurrence cur[j] = min(t[j], cur[j - 1] + 1) is a running minimum of t[j] - j."""
    pats, txts = [p for p, _ in pairs], [t for _, t in pairs]
    m = np.array([len(p) for p in pats])
    tl = np.array([len(t) for t in txts])
    M, T = int(m.max()), int(tl.max())
    pat, txt = _codes(pats, M, 99)[:, :M], _codes(txts, T, 98)
    ar = np.arange(M + 1)
    prev = np.tile(ar, (len(pairs), 1))
    d = m.copy()  # an empty text: the pattern is empty too
    for i in range(1, T + 1):
        t = np.empty_like(prev)
        t[:, 0] = i
        t[:, 1:] = np.minimum(prev[:, 1:] + 1, prev[:, :-1] + (txt[:, i - 1:i] != pat))
        cur = np.minimum.accumulate(t - ar, axis=1) + ar
        sel = tl == i
        d[sel] = cur[sel, m[sel]]
        prev = cur
    return d


_DIST = {}


def _key(a, b):
    return (a, b) if (len(a), a) <= (len(b), b) else (b, a)


def distances(pairs):
    """{(pattern, text): edit distance} for every pair, cached per distinct pair (pattern = the shorter string)."""
    want = sorted({_key(a, b) for a, b in pairs if a != b} - _DIST.keys())
    for batch in _batches(want):
        for pt, d in zip(batch, dp_distances(batch)):
            _DIST[pt] = int(d)
    return _DIST


def sim(a, b):
    """levenshtein_similarity: 1 - d / max_len floored at 1e-8; identical strings (two empty ones too) 1.0."""
    if a == b:
        return 1.0
    return max(FLOOR, 1 - _DIST[_key(a, b)] / max(len(a), len(b)))


def matrix(group):
    k = len(group)
    M = np.full((k, k), np.nan)
    for i in range(k):
        for j in range(k):
            if i != j:
                M[i, j] = sim(group[i], group[j])
    return M


def brute(groups):
    """(best index int32 [G], mean float64 [G]): np.nanmean over the rows of the matrix with a NaN diagonal, np.argmax."""
    distances([(a, b) for g in groups for a in set(g) for b in set(g)])
    idx, avg = np.zeros(len(groups), np.int32), np.zeros(len(groups))
    for g, grp in enumerate(groups):
        means = np.nanmean(matrix(grp), axis=1)
        idx[g] = int(np.argmax(means))
        avg[g] = means[idx[g]]
    return idx, avg


# ----------------------------------------------------------------------------- medoid_kernel restated

MUTATIONS = ("32-bit word up to m = 40", "ph <<= 1 without | 1", "sequential row sum", "diagonal skipped", ">= for the lane maximum",
             "highest index wins a cross-lane tie", "no floor", "classes from the key without confirming the characters")


_MYERS = {}


def myers_distances(pairs, word32_max=32, seed_or=True):
    """myers<W> of (pattern, text) pairs, 0 < len(pattern) <= 64: W = uint32 for patterns up to word32_max characters (the
    64-bit match table cast to it), uint64 above; the score reads bit m - 1; `seed_or`: ph = (ph << 1) | 1.  Cached per
    pair, word and seed."""
    key = lambda p, t: (len(p) <= word32_max, seed_or, p, t)  # noqa: E731
    todo = sorted({(p, t) for p, t in pairs if key(p, t) not in _MYERS})
    for batch in _batches(todo):
        P = len(batch)
        m = np.array([len(p) for p, _ in batch], np.uint64)
        tl = np.array([len(t) for _, t in batch])
        mask = np.where(m <= word32_max, np.uint64(0xFFFFFFFF), np.uint64(0xFFFFFFFFFFFFFFFF))
        peq = np.zeros((P, 37), np.uint64)  # symbol 36: past the end of a text, matches nothing
        for r, (p, _) in enumerate(batch):
            for q, c in enumerate(_codes([p], len(p), 0)[0]):
                peq[r, c] |= np.uint64(1 << q)
        peq &= mask[:, None]
        txt = _codes([t for _, t in batch], int(tl.max()), 36)
        rows = np.arange(P)
        one, seed = np.uint64(1), np.uint64(1 if seed_or else 0)
        pv, mv = mask.copy(), np.zeros(P, np.uint64)
        score = m.astype(np.int64)
        sh = m - one
        for k in range(int(tl.max())):
            eq = peq[rows, txt[:, k]]
            xv = eq | mv
            xh = ((((eq & pv) + pv) & mask) ^ pv) | eq
            ph = mv | (~(xh | pv) & mask)
            mh = pv & xh
            step = ((ph >> sh) & one).astype(np.int64) - ((mh >> sh) & one).astype(np.int64)
            score += np.where(k < tl, step, 0)
            ph = ((ph << one) | seed) & mask
            mh = (mh << one) & mask
            pv = mh | (~(xv | ph) & mask)
            mv = ph & xv
        _MYERS.update(zip([key(p, t) for p, t in batch], score.tolist()))
    return {(p, t): _MYERS[key(p, t)] for p, t in pairs}


def np_sum(xs):
    """numpy's DOUBLE_pairwise_sum for n <= 128 (kc_numeric.cuh np_sum): below 8 terms one by one from -0.0, else 8
    accumulators, ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), the tail one by one; then + 0.0."""
    n = len(xs)
    if n < 8:
        res = -0.0
        for x in xs:
            res += x
    else:
        r = list(xs[:8])
        i, n8 = 8, n - n % 8
        while i < n8:
            for q in range(8):
                r[q] += xs[i + q]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for x in xs[i:]:
            res += x
    return 0.0 + res


def fnv1a(s):
    h = 2166136261
    for c in s.encode():
        h = ((h ^ c) * 16777619) & 0xFFFFFFFF
    return h


def classes(group, mutation=None):
    """s_rep of every string: for k <= 32 the lowest lane with the same (hash, length) key, kept only if every lane's
    characters confirm it (__all_sync), else (and for k > 32) the first identical string by the exact scan."""
    k = len(group)
    h, L = [fnv1a(s) for s in group], [len(s) for s in group]
    if k <= 32:
        first = {}
        rep = [first.setdefault(h[i] ^ ((L[i] * 0x9E3779B1) & 0xFFFFFFFF), i) for i in range(k)]
        confirm = mutation != MUTATIONS[7]
        if all(rep[i] == i or not confirm or group[rep[i]] == group[i] for i in range(k)):
            return rep
    return [next(j for j in range(i + 1) if h[j] == h[i] and L[j] == L[i] and group[j] == group[i]) for i in range(k)]


def _class_pairs(group, mutation=None):
    """(class of every string, the class representatives, the (a, b) class pairs with their pattern and text)."""
    rep = classes(group, mutation)
    uniq = [i for i in range(len(group)) if rep[i] == i]
    num = {i: c for c, i in enumerate(uniq)}
    cls = [num[rep[i]] for i in range(len(group))]
    pairs = []
    for a in range(len(uniq)):
        for b in range(a + 1, len(uniq)):
            pa, ta = (b, a) if len(group[uniq[a]]) > len(group[uniq[b]]) else (a, b)
            pairs.append((a, b, group[uniq[pa]], group[uniq[ta]]))
    return cls, uniq, pairs


def restated(groups, mutation=None):
    """medoid_kernel<4> under method 0 for every group, optionally with one of MUTATIONS: (index int32 [G], mean float64 [G])."""
    word32_max = 40 if mutation == MUTATIONS[0] else 32
    seed_or = mutation != MUTATIONS[1]
    per_group = [_class_pairs(g, mutation) for g in groups]
    need = {(p, t) for _, _, pairs in per_group for _, _, p, t in pairs if p}
    dist = myers_distances(sorted(need), word32_max, seed_or)
    idx, avg = np.zeros(len(groups), np.int32), np.zeros(len(groups))
    for g, (grp, (cls, uniq, pairs)) in enumerate(zip(groups, per_group)):
        k, u = len(grp), len(uniq)
        S = [[1.0] * u for _ in range(u)]
        for a, b, p, t in pairs:
            d = dist[(p, t)] if p else len(t)
            sv = 1.0 - d / len(t)
            S[a][b] = S[b][a] = sv if mutation == MUTATIONS[6] else (sv if sv > FLOOR else FLOOR)
        lanes = [(-1.0, 0x7FFFFFFF)] * 32
        for i in range(k):
            row = [0.0 if j == i else S[cls[i]][cls[j]] for j in range(k)]
            if mutation == MUTATIONS[2]:
                tot = 0.0
                for x in row:
                    tot += x
            elif mutation == MUTATIONS[3]:
                tot = np_sum(row[:i] + row[i + 1:])
            else:
                tot = np_sum(row)
            a = tot / (k - 1)
            mine = lanes[i % 32][0]
            if a > mine or (mutation == MUTATIONS[4] and a == mine):
                lanes[i % 32] = (a, i)
        for st in (16, 8, 4, 2, 1):
            nxt = []
            for ln in range(32):
                (ma, mi), (oa, oi) = lanes[ln], lanes[ln ^ st]
                lower = oi > mi if mutation == MUTATIONS[5] else oi < mi
                nxt.append((oa, oi) if oa > ma or (oa == ma and lower) else (ma, mi))
            lanes = nxt
        avg[g], idx[g] = lanes[0]
    return idx, avg


# ----------------------------------------------------------------------------- the edge families


def rand_str(r, n, alphabet=ALNUM):
    return "".join(r.choice(alphabet) for _ in range(n))


def variant(r, s, edits, alphabet=ALNUM):
    """s with `edits` random substitutions, insertions or deletions."""
    s = list(s)
    for _ in range(edits):
        op = r.randrange(3) if s else 1
        if op == 0:
            s[r.randrange(len(s))] = r.choice(alphabet)
        elif op == 1:
            s.insert(r.randrange(len(s) + 1), r.choice(alphabet))
        else:
            del s[r.randrange(len(s))]
    return "".join(s)


def word_pair(r, m, tl, style):
    """A pattern of m characters and a different text of tl >= m characters in one of five styles: random; one letter (the
    carry of (eq & pv) + pv runs through the whole word); two letters; the pattern's only match at bit m - 1; a text that
    starts with the pattern."""
    if style == "random":
        p, t = rand_str(r, m), rand_str(r, tl)
    elif style == "one letter":
        p = "a" * m
        t = "".join("b" if r.random() < 0.1 else "a" for _ in range(tl))
    elif style == "two letters":
        p, t = rand_str(r, m, "ab"), rand_str(r, tl, "ab")
    elif style == "top bit":
        p = "b" * (m - 1) + "a"
        t = rand_str(r, tl, "acdefg")
    else:
        p = rand_str(r, m)
        t = p + rand_str(r, tl - m)
    if t == p:
        t = t[:-1] + ("z" if t[-1] != "z" else "y")
    return p, t


STYLES = ("random", "one letter", "two letters", "top bit", "prefix")


def fam_word(r):
    """Patterns of 1, 31, 32, 33, 63 and 64 characters against texts of m, m + 1, 65, 200 and 2000, in every style; groups
    of up to 64 add variants of the pattern (at most 64 characters) around the pair, at random positions."""
    groups = []
    for m in PATTERN_LENGTHS:
        for tl in sorted({m, m + 1, 65, 200, 2000}):
            for style in STYLES:
                p, t = word_pair(r, m, tl, style)
                grp = [p, t]
                if tl <= 200:
                    grp += [variant(r, p, r.randint(1, 3), "ab" if style in ("one letter", "two letters") else ALNUM)[:64]
                            for _ in range(r.choice([0, 1, 3, 7, 40]))]
                r.shuffle(grp)
                groups.append(grp)
    return groups


def fam_choice(r):
    """Equal-length distinct strings (the pattern is the lower class at equal lengths), and 64-string groups whose one string
    longer than 64 characters sits at index 0, 31, 32 or 63."""
    groups = []
    for L in (1, 2, 17, 31, 32, 33, 63, 64):
        for k in (2, 3, 6, 33):
            base = rand_str(r, L)
            grp = [base]
            while len(grp) < k:
                s = list(rand_str(r, L) if r.random() < 0.2 else base)
                for _ in range(r.randint(1, 3)):
                    s[r.randrange(L)] = r.choice(ALNUM[:4] if L < 3 else ALNUM)
                grp.append("".join(s))
            groups.append(grp)
    for pos in (0, 31, 32, 63):
        for long_len in (65, 200, 2000):
            base = rand_str(r, 40)
            grp = [variant(r, base, r.randint(0, 30))[:64] for _ in range(64)]
            grp[pos] = base + rand_str(r, long_len - 40)
            groups.append(grp)
    return groups


def fam_empty(r):
    """Empty strings against non-empty ones (d = tl), groups of empty strings only, and disjoint strings of equal or unequal
    length (similarity 0, lifted to the 1e-8 floor)."""
    groups = []
    for k in (2, 3, 5, 32, 33, 64):
        groups.append([""] * k)
        grp = ["" if r.random() < 0.4 else rand_str(r, r.choice([1, 5, 32, 33, 64])) for _ in range(k)]
        grp[r.randrange(k)] = ""
        groups.append(grp)
    for L in (1, 3, 8, 31, 32, 33, 64):
        for k in (2, 4, 9, 33):
            alphabets = ["abcdefghi", "jklmnopqr", "stuvwxyz0", "123456789"]
            grp = [rand_str(r, L if r.random() < 0.7 else r.randint(1, 64), alphabets[r.randrange(4)]) for _ in range(k)]
            if r.random() < 0.3:
                grp[r.randrange(k)] = ""
            groups.append(grp)
    return groups


def fam_classes(r, collision):
    """u = 1; u = k = 64 (all 2016 pairs); u = 33 (both ballots); a duplicate whose first copy is at index 32 or more; an
    FNV-1a collision pair in groups of 32 or fewer (the __all_sync fall-back) and of more than 32."""
    groups = []
    for k in (2, 5, 31, 32, 33, 63, 64):
        groups.append([rand_str(r, r.choice([1, 7, 40]))] * k)
    for _ in range(4):
        base = rand_str(r, r.randint(6, 14))
        grp = set()
        while len(grp) < 64:
            grp.add(variant(r, base, r.randint(1, 5)))
        grp = sorted(grp)
        r.shuffle(grp)
        groups.append(grp)
    for k in (33, 40, 64, 64):
        base = rand_str(r, 10)
        distinct = set()
        while len(distinct) < 33:
            distinct.add(variant(r, base, r.randint(1, 4)))
        distinct = sorted(distinct)
        r.shuffle(distinct)
        grp = distinct + [r.choice(distinct) for _ in range(k - 33)]
        r.shuffle(grp)
        groups.append(grp)
    for k in (34, 40, 50, 64, 64, 64):
        base = rand_str(r, 12)
        grp = [variant(r, base, r.randint(1, 4)) for _ in range(k)]
        first = r.randint(32, k - 2)
        grp[first] = variant(r, base, 6)
        for i in r.sample(range(first + 1, k), r.randint(1, min(3, k - first - 1))):
            grp[i] = grp[first]
        groups.append(grp)
    a, b = collision
    for k in (2, 3, 8, 31, 32, 33, 40, 64):
        for _ in range(3):
            grp = [variant(r, a, r.randint(1, 4)) if r.random() < 0.6 else rand_str(r, 8) for _ in range(k)]
            i, j = r.sample(range(k), 2)
            grp[i], grp[j] = a, b
            if k > 2 and r.random() < 0.5:
                grp[r.choice([x for x in range(k) if x not in (i, j)])] = r.choice([a, b])
            groups.append(grp)
    return groups


def fam_ties(r):
    """Exact ties of the best mean: copies of a centre string among its variants of the same power-of-two length (every
    similarity is a multiple of 1 / L, so every row sum is exact whatever the order), each variant at most once or twice.
    The centre's copies sit at rows i and i + 32 (one lane), or on different lanes, or both."""
    groups = []
    for _ in range(60):
        L = r.choice([8, 16, 32, 64])
        A = rand_str(r, L)
        kind = r.choice(["same lane", "same lane", "other lane", "both"])
        k = r.randint(34, 64) if kind != "other lane" else r.choice([r.randint(3, 32), r.randint(33, 64)])
        pool = set()
        while len(pool) < max(2, k // 2):
            s = list(A)
            for q in r.sample(range(L), r.randint(1, 2)):
                s[q] = r.choice(ALNUM)
            s = "".join(s)
            if s != A:
                pool.add(s)
        grp = sorted(pool) * 2
        r.shuffle(grp)
        grp = grp[:k]
        if kind == "same lane":
            i = r.randint(0, k - 33)
            at = [i, i + 32]
        elif kind == "other lane":
            at = r.sample(range(k), 2)
            while (at[0] - at[1]) % 32 == 0:
                at = r.sample(range(k), 2)
        else:
            i = r.randint(0, k - 33)
            at = [i, i + 32, r.choice([x for x in range(k) if (x - i) % 32])]
        for i in at:
            grp[i] = A
        groups.append(grp)
    return groups


def _winners(S, cls):
    """The winner of a class-structured group by numpy (nanmean, argmax), by a sequential row sum and with the diagonal
    skipped."""
    k = len(cls)
    M = S[np.ix_(cls, cls)]
    np.fill_diagonal(M, np.nan)
    ref = int(np.argmax(np.nanmean(M, axis=1)))
    Z = np.where(np.isnan(M), 0.0, M)
    seq = int(np.argmax(np.cumsum(Z, axis=1)[:, -1] / (k - 1)))
    off = M[~np.eye(k, dtype=bool)].reshape(k, k - 1)
    skip = int(np.argmax(np.sum(off, axis=1) / (k - 1)))
    return ref, seq, skip


def fam_order(r, want=50):
    """Groups of k >= 9 classes of identical strings (pairs either disjoint, at the floor, or near) whose numpy winner differs
    from the winner under a sequential row sum or with the diagonal skipped; found by search."""
    found = {"sequential": [], "skipped": []}
    while min(len(v) for v in found.values()) < want:
        cands = []
        for _ in range(150):
            ncls = r.randint(2, 8)
            strs = set()
            while len(strs) < ncls:
                strs.add(variant(r, rand_str(r, r.choice([7, 11, 13]), "abcdefg"), r.randint(0, 3), "abcdefg")
                         if r.random() < 0.6 else rand_str(r, r.choice([5, 9, 13]), "hijklmnopqrstuvwxyz"))
            strs = sorted(strs)
            k = r.randint(9, 64)
            cls = [r.randrange(ncls) for _ in range(k)]
            cands.append((strs, cls))
        distances([(a, b) for strs, _ in cands for a in strs for b in strs])
        for strs, cls in cands:
            S = np.array([[sim(a, b) for b in strs] for a in strs])
            ref, seq, skip = _winners(S, cls)
            grp = [strs[c] for c in cls]
            if seq != ref and len(found["sequential"]) < want:
                found["sequential"].append(grp)
            elif skip != ref and len(found["skipped"]) < want:
                found["skipped"].append(grp)
    return found["sequential"] + found["skipped"]


_FAMS = {}


def families(seed=0):
    """{family: groups}, built once per seed."""
    if seed not in _FAMS:
        r = random.Random(seed)
        collision = _fnv_collision()
        _FAMS[seed] = {"word": fam_word(r), "choice": fam_choice(r), "empty": fam_empty(r), "classes": fam_classes(r, collision),
                       "ties": fam_ties(r), "order": fam_order(r)}
        for grps in _FAMS[seed].values():
            for g in grps:
                assert 2 <= len(g) <= 64 and sum(len(s) > 64 for s in g) <= 1 and max(map(len, g)) <= 2000
                assert all(set(s) <= set(ALNUM) for s in g)
    return _FAMS[seed]


def all_groups(seed=0):
    return [g for f in FAMILIES for g in families(seed)[f]]


# ----------------------------------------------------------------------------- counts behind the floors


def counts(seed=0):
    """What the families reach, counted on the host from the brute force."""
    fams = families(seed)
    distances([(x, y) for grps in fams.values() for g in grps for x in set(g) for y in set(g)])
    c = collections.Counter()
    a, b = _fnv_collision()
    for f, grps in fams.items():
        for g in grps:
            u = len(set(g))
            for x, y in {_key(x, y) for x in set(g) for y in set(g) if x != y}:
                m, tl = len(x), len(y)
                c["pairs with m in {32, 33, 64}"] += m in (32, 33, 64)
                c["pairs with m in {31, 32, 33, 63, 64}, tl >= 200"] += m in (31, 32, 33, 63, 64) and tl >= 200
                c["pairs with an empty pattern"] += m == 0 < tl
                c["equal-length pairs"] += m == tl
                c["pairs at the floor"] += sim(x, y) == FLOOR
                c["equal-length pairs at the floor"] += sim(x, y) == FLOOR and m == tl
            c["u = 1"] += u == 1
            c["u = k = 64"] += u == len(g) == 64
            c["u = 33"] += u == 33
            c["duplicate first seen at 32 or more"] += any(g.index(s) >= 32 and g.count(s) > 1 for s in set(g))
            c["collision, k <= 32"] += a in g and b in g and len(g) <= 32
            c["collision, k > 32"] += a in g and b in g and len(g) > 32
            c["long string at 0, 31, 32, 63 of 64"] += len(g) == 64 and any(len(g[p]) > 64 for p in (0, 31, 32, 63))
            means = np.nanmean(matrix(g), axis=1)
            at = np.flatnonzero(means == means.max())
            c["ties of rows i and i + 32"] += any((j - i) % 32 == 0 for i in at for j in at if j > i)
            c["ties across lanes"] += any((j - i) % 32 != 0 for i in at for j in at if j > i)
        if f == "order":
            c["groups the summation order decides"] += len(grps)
    return c


FLOORS = {"pairs with m in {32, 33, 64}": 250, "pairs with m in {31, 32, 33, 63, 64}, tl >= 200": 50, "pairs with an empty pattern": 40,
          "equal-length pairs": 300, "pairs at the floor": 300, "equal-length pairs at the floor": 60, "u = 1": 7,
          "u = k = 64": 4, "u = 33": 4, "duplicate first seen at 32 or more": 6, "collision, k <= 32": 12, "collision, k > 32": 8,
          "long string at 0, 31, 32, 63 of 64": 12, "ties of rows i and i + 32": 30, "ties across lanes": 25,
          "groups the summation order decides": 100}


# ----------------------------------------------------------------------------- the alignment pre-pass's string pairs

ALIGN_PATTERNS = (31, 32, 33, 49, 50)


def align_nodes(seed=0):
    """List nodes of strings for kc_debug_alignsim_nodes: patterns of 31, 32, 33, 49 and 50 characters (at most 50 raw
    characters, so every pair with one is decided) in every style against texts of m + 1, 65, 200 and 2000 characters,
    with variants of the pattern; a node may hold two long texts (that pair is left NaN)."""
    r = random.Random(seed)
    nodes = []
    for m in ALIGN_PATTERNS:
        for tl in (m + 1, 65, 200, 2000):
            for style in STYLES:
                p, t = word_pair(r, m, tl, style)
                node = [p, t] + [variant(r, p, r.randint(1, 3))[:50] for _ in range(r.choice([0, 2, 5]))]
                if r.random() < 0.3:
                    node.append(t[:-1] + "0")
                r.shuffle(node)
                nodes.append(node)
    return nodes


def align_expected(nodes):
    """1 - d / longest floored at 1e-8 for every pair a < b; 1.0 for identical strings; NaN on the diagonal and where both
    strings are longer than 50 characters."""
    distances([(a, b) for nd in nodes for a in nd for b in nd])
    parts = []
    for nd in nodes:
        T = len(nd)
        E = np.full((T, T), np.nan)
        for i in range(T):
            for j in range(T):
                if i != j and not (len(nd[i]) > 50 and len(nd[j]) > 50):
                    E[i, j] = sim(nd[i], nd[j])
        parts.append(E.reshape(-1))
    return np.concatenate(parts)


def run_align(nodes, device=-1, lanes=1):
    from k_llms_b200 import _native as K
    flat = [json.dumps(s).encode() for nd in nodes for s in nd]
    texts = (ctypes.c_char_p * len(flat))(*flat)
    lens = np.array([len(nd) for nd in nodes], dtype=np.int32)
    out = np.full(int((lens.astype(np.int64) ** 2).sum()), 0x7FF4DEAD0000BEEF, dtype=np.uint64).view(np.float64)
    rc = K.load().kc_debug_alignsim_nodes(ctypes.cast(texts, ctypes.c_void_p), lens.ctypes.data, len(nodes), lanes, device, out.ctypes.data)
    if rc < 0:
        K.check(rc)
    return out


# ----------------------------------------------------------------------------- JSON records


def _raw(r, s, multi):
    """A raw spelling of normalised s: upper-case letters and punctuation the normalisation drops, three words when
    `multi` (and s has three to 48 characters); at most 50 characters when s has at most 50."""
    out = "".join(c.upper() if r.random() < 0.2 else c for c in s)
    if multi and 3 <= len(s) <= 48:
        q, w = sorted(r.sample(range(1, len(s)), 2))
        out = out[:q] + " " + out[q:w] + " " + out[w:]
    if len(out) < 50 and r.random() < 0.3:
        out += r.choice(",.!")
    return out if len(s) > 50 or len(out) <= 50 else s


def json_groups():
    """Edge groups whose strings fit the JSON paths' rule: at most one longer than 50 raw characters; from the word-size
    edges with patterns of 31, 32, 33, 49 and 50 characters (the alignment nodes), and the empty, class and tie families."""
    fams = families()
    groups = [nd for seed in (1, 2) for nd in align_nodes(seed) if sum(len(s) > 50 for s in nd) <= 1]
    groups += [g for f in ("empty", "classes", "ties") for g in fams[f] if sum(len(s) > 50 for s in g) <= 1]
    return groups


def json_records(groups, seed=0):
    """{n: (records, groups)}: one record per group, its strings in field "s" beside a constant field "k".  A string of
    three or more words makes the field a similarity medoid (cu:1405-1411); a long string is cut into words of nine
    characters."""
    r = random.Random(seed)
    out = {}
    for g in groups:
        raws = []
        for i, s in enumerate(g):
            if len(s) > 50:
                raws.append(" ".join(s[q:q + 9] for q in range(0, len(s), 9)))
            else:
                raws.append(_raw(r, s, multi=(i == 0 or r.random() < 0.5)))
        if not any(len(x.split()) >= 3 for x in raws):
            continue
        texts = [json.dumps({"k": 1, "s": x}) for x in raws]
        recs, grps = out.setdefault(len(g), ([], []))
        recs.append(texts)
        grps.append(g)
    return out


# ----------------------------------------------------------------------------- tests


def test_dp_matches_python_and_native_edit_distances():
    """The batched DP against oracle.consensus_py.edit_distance on a sample of the families' pairs and against
    kc_levenshtein on every pair."""
    from k_llms_b200 import _native as K
    groups = all_groups() + align_nodes()
    dist = distances([(a, b) for g in groups for a in set(g) for b in set(g)])
    pairs = sorted({_key(a, b) for g in groups for a in set(g) for b in set(g) if a != b})
    bad = [(p, t) for p, t in pairs if K.levenshtein(p, t) != dist[(p, t)]]
    assert not bad, (len(bad), bad[:3])
    r = random.Random(3)
    sample = r.sample([pt for pt in pairs if len(pt[1]) <= 200], 600) + r.sample([pt for pt in pairs if len(pt[1]) > 200], 12)
    bad = [(p, t) for p, t in sample if edit_distance(p, t) != dist[(p, t)]]
    assert not bad, (len(bad), bad[:3])
    print(f"\n{len(pairs)} distinct pairs against kc_levenshtein, {len(sample)} against edit_distance")


def test_brute_force_matches_c_oracle():
    """ko_medoid_str on every group of every family: the same index and the same mean bits."""
    for f in FAMILIES:
        groups = families()[f]
        idx, avg = brute(groups)
        oi, oa = OC.medoid(groups)
        assert np.array_equal(oi, idx), (f, np.flatnonzero(oi != idx)[:5])
        assert np.array_equal(oa.view(np.uint64), avg.view(np.uint64)), f


def test_restatement_equals_brute_force():
    """The restated medoid_kernel (classes as the kernel forms them, Myers in 32- and 64-bit words, np_sum, the lane maximum
    and the shuffle) equals the brute force on every family, index and mean bits."""
    for f in FAMILIES:
        groups = families()[f]
        idx, avg = brute(groups)
        ri, ra = restated(groups)
        bad = np.flatnonzero((ri != idx) | (ra.view(np.uint64) != avg.view(np.uint64)))
        assert not bad.size, (f, bad[:5], [(ri[g], ra[g], idx[g], avg[g]) for g in bad[:3]])


def test_myers_restatement_at_every_pattern_length():
    """Myers with the kernel's word choice equals the DP at every pattern length from 1 to 64 against texts of m to 2000
    characters, in every style."""
    r = random.Random(9)
    pairs = [word_pair(r, m, tl, style) for m in range(1, 65) for tl in {m, m + 1, 65, r.randint(m, 300), 2000} for style in STYLES]
    dist = distances(pairs)
    got = myers_distances(pairs)
    bad = [pt for pt in pairs if got[pt] != dist[_key(*pt)]]
    assert not bad, (len(bad), bad[:2])


def test_mutated_restatement_goes_wrong_on_the_families():
    """Each mutation of the restatement gets groups wrong (index or mean bits), and the families it is built against catch
    it: the word-size edges a 32-bit word up to m = 40 and a top row seeded without | 1; the order-sensitive groups a
    sequential sum and a skipped diagonal; the ties the lane and cross-lane tie rules; the floor groups a missing floor; the
    FNV-1a collision in groups of 32 or fewer the missing character confirmation."""
    caught = {MUTATIONS[0]: "word", MUTATIONS[1]: "word", MUTATIONS[2]: "order", MUTATIONS[3]: "order", MUTATIONS[4]: "ties",
              MUTATIONS[5]: "ties", MUTATIONS[6]: "empty", MUTATIONS[7]: "classes"}
    wrong = collections.defaultdict(collections.Counter)
    for f in FAMILIES:
        groups = families()[f]
        idx, avg = brute(groups)
        for mutation in (None,) + MUTATIONS:
            ri, ra = restated(groups, mutation)
            wrong[mutation][f] += int(((ri != idx) | (ra.view(np.uint64) != avg.view(np.uint64))).sum())
    print("\ngroups each mutation gets wrong:", {m: dict(c) for m, c in wrong.items()})
    assert sum(wrong[None].values()) == 0, dict(wrong[None])
    for mutation, fam in caught.items():
        assert wrong[mutation][fam] >= 5, (mutation, dict(wrong[mutation]))


def test_collision_pair_shares_the_kernels_key():
    """The collision pair is two different strings of one length with one FNV-1a hash (the vectorised helper and the
    restatement's), so that __match_any_sync gives them one (hash, length) key."""
    a, b = _fnv_collision()
    h = _fnv1a(np.frombuffer((a + b).encode(), np.uint8).reshape(2, 8))
    assert a != b and len(a) == len(b) and h[0] == h[1] == fnv1a(a) == fnv1a(b)
    assert classes([a, b]) == [0, 1] and classes([a, b], MUTATIONS[7]) == [0, 0]


def test_floors():
    c = counts()
    print("\n" + "; ".join(f"{k}: {v}" for k, v in sorted(c.items())))
    low = {k: (c[k], v) for k, v in FLOORS.items() if c[k] < v}
    assert not low, low


def test_alignsim_host_phase_on_the_edge_nodes():
    """The alignment pre-pass's similarity phase, instantiated on the host with one lane and with 32: every decided pair
    equals 1 - d / longest (floored), NaN exactly on the diagonal and between two strings longer than 50 characters."""
    nodes = align_nodes()
    exp = align_expected(nodes)
    for lanes in (1, 32):
        assert_matrices(run_align(nodes, -1, lanes), exp)


def test_json_paths_with_the_oracle_pick_the_brute_force_medoid():
    """The edge groups as JSON records: the device JSON path's phases on the host (jsongpu_with_oracle) and H1 with the C
    oracle (consolidate_json_with_oracle) take every record and print the brute force's medoid string."""
    from tests.helpers import consolidate_json_with_oracle, jsongpu_with_oracle
    total = long_pairs = 0
    for n, (records, groups) in sorted(json_records(json_groups()).items()):
        idx, _ = brute(groups)
        dev, status = jsongpu_with_oracle(records)
        h1 = consolidate_json_with_oracle(records)
        for r, texts in enumerate(records):
            want = json.loads(texts[idx[r]])["s"]
            assert status[r] == 0 and json.loads(dev[r][0])["s"] == want, (n, r, status[r], dev[r], want)
            assert h1[r] is not None and json.loads(h1[r][0])["s"] == want, (n, r, h1[r], want)
            total += 1
            long_pairs += any(len(s) > 64 for s in groups[r]) and any(len(s) in ALIGN_PATTERNS for s in groups[r])
    print(f"\n{total} records, {long_pairs} with a pattern of 31, 32, 33, 49 or 50 characters and a text longer than 64")
    assert total >= 200 and long_pairs >= 80, (total, long_pairs)
