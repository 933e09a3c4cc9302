"""Shared test helpers: golden loading, strict equality (float bits, key order), a CPU stand-in device, which kernels ran."""
import contextlib
import json
import math
import os
import re

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    with open(os.path.join(GOLDEN, name + ".json")) as f:
        return json.load(f)["cases"]


def same(a, b) -> bool:
    """Equality the way the parity bar means it: same types, same dict key ORDER, same float bits (NaN == NaN)."""
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))
    if type(a) is not type(b):
        return False
    if isinstance(a, dict):
        return list(a) == list(b) and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return a == b


def random_codes(rng, G, n, vocab, p_none=0.08, p_absent=0.03, p_agree=0.6):
    """K1 input: int32 [G, n] codes around a per-group truth, with None (-1) and absent (-2) cells."""
    truth = rng.integers(0, vocab, (G, 1))
    draw = rng.integers(0, vocab, (G, n))
    codes = np.where(rng.random((G, n)) < p_agree, truth, draw).astype(np.int32)
    codes[rng.random((G, n)) < p_none] = -1
    codes[rng.random((G, n)) < p_absent] = -2
    return codes


def random_vals(rng, G, n, style):
    """K2 input: float64 [G, n] in one of five styles, with None / absent / NaN / inf cells."""
    from oracle.columnar import F64_ABSENT, F64_NONE
    if style == "ints":
        t = np.floor(rng.random((G, 1)) * 1e6) + 1
        d = np.floor(rng.random((G, n)) * 1e6) + 1
    elif style == "near":  # straddle the 3% tolerance, both signs, zeros, tiny values
        base = rng.choice([1.0, -1.0, 100.0, 1e-7, 0.0, 12.5, -3000.0], (G, 1))
        t = base
        d = base * (1.0 + rng.choice([-0.05, -0.031, -0.029, 0.0, 0.015, 0.0299, 0.0301, 0.06], (G, n)))
    elif style == "pow10":  # decimal-shift and sign mistakes -> tie-resolution paths
        base = rng.choice([12.5, 7.0, 0.125, 3.3], (G, 1))
        t = base
        d = base * rng.choice([1.0, 10.0, 0.1, -1.0, 100.0, 1.0, 1.0], (G, n))
    elif style == "lowbits":  # values that differ only in low mantissa bits (32-bit sort keys tie; repair path)
        base = rng.choice([1.0, -1.0, 3.141592653589793, 1e-300, -7e5, 123456.0], (G, 1))
        t = base
        d = base * (1.0 + rng.integers(-40, 40, (G, n)) * 2.0 ** rng.choice([-52, -50, -45, -40, -33, -30, -20], (G, 1)))
    else:
        t = rng.uniform(1, 1e4, (G, 1))
        d = rng.uniform(1, 1e4, (G, n))
    p_agree = rng.choice([0.2, 0.5, 0.8], (G, 1))
    vals = np.where(rng.random((G, n)) < p_agree, t, d).astype(np.float64)
    vals[rng.random((G, n)) < 0.08] = F64_NONE
    vals[rng.random((G, n)) < 0.03] = F64_ABSENT
    vals[rng.random((G, n)) < 0.02] = np.nan
    vals[rng.random((G, n)) < 0.01] = np.inf
    return np.ascontiguousarray(vals)


VAL_STYLES = ("ints", "near", "pow10", "floats", "lowbits")

# (rel_eps, abs_eps) settings that put K2's tolerance tests on their edges: the default, exact equality, very loose, and
# a relative tolerance below one ulp with a denormal absolute one
EDGE_EPS = ((0.03, 1e-6), (0.0, 0.0), (0.9, 10.0), (1e-12, 1e-300))


def numeric_edge_vals(rng, G, n):
    """K2 input where the majority shortcut has to give up or sits on a boundary, and the general kernels' tie and low-bit
    repair paths run: neighbours right at the tolerance, cells sharing v's high word, signed zeros, -inf / negative NaN /
    odd NaN payloads, absent cells, overflow of the sum, every majority size."""
    from oracle.columnar import F64_ABSENT, F64_NONE
    pool = np.array([0.0, -0.0, 1.0, 5e-324, 1e-310, 2.0 ** -1022, 1.7e308, 9e307, 123456.0, 0.1, 1e15 + 0.5, 3.0, 2.0 ** 52,
                     1048576.0, 1048577.0, 0.999999, 33.333333333333336], dtype=np.float64)
    v = pool[rng.integers(0, len(pool), G)]
    odd = np.array([F64_NONE, F64_ABSENT, np.nan, -np.nan, np.inf, -np.inf], dtype=np.float64)
    odd = np.concatenate([odd, np.array([0x7FFFFFFFFFFFFFFF, 0xFFF8000000000001, 0x7FF8C0DE00000001, 0x7FF8C0E000000000],
                                        dtype=np.uint64).view(np.float64)])
    factor = np.array([0.97, 0.9700000001, 0.9699999999, 1.03, 1.0300000001, 1.0299999999, 1 + 1e-9, 1 - 2.0 ** -20, 1 + 2.0 ** -21,
                       1 + 2.0 ** -33, 0.5, 2.0, -1.0, 1.0309278350515465, 0.9708737864077669], dtype=np.float64)
    vals = np.repeat(v[:, None], n, axis=1)
    c = rng.integers(1, n + 1, G)                                  # copies of v kept
    for g in range(G):
        k = n - c[g]
        if k == 0:
            continue
        pos = rng.choice(n, k, replace=False)
        kind = rng.integers(0, 5, k)
        repl = np.where(kind == 0, odd[rng.integers(0, len(odd), k)],
                np.where(kind == 1, v[g] * factor[rng.integers(0, len(factor), k)],
                np.where(kind == 2, np.nextafter(v[g], np.inf * rng.choice([-1.0, 1.0], k)),
                np.where(kind == 3, F64_NONE, rng.uniform(-10, 2e6, k)))))
        vals[g, pos] = repl
    return np.ascontiguousarray(vals)


def _up(x, k=1):
    """The float k ulps above x."""
    for _ in range(k):
        x = math.nextafter(x, math.inf)
    return x


def _down(x, k=1):
    """The float k ulps below x."""
    for _ in range(k):
        x = math.nextafter(x, -math.inf)
    return x


def raising_embeddings(texts):
    raise RuntimeError("no network in tests")


# ----------------------------------------------------------------------------- exact number conversions (kc_jsoncore.cuh)

def number_texts():
    """JSON number texts for to_double: random floats, 19-digit ints, fixed and exponent notation, a few known hard cases."""
    import random
    rng = random.Random(5)
    texts = [repr(rng.random() * 1e4 + 1) for _ in range(20000)]
    texts += [str(rng.randrange(-10 ** 19, 10 ** 19)) for _ in range(20000)]
    texts += ["%.*f" % (rng.randrange(0, 12), rng.random() * 10 ** rng.randrange(-3, 9)) for _ in range(20000)]
    texts += ["%.*e" % (rng.randrange(0, 18), rng.random() * 10.0 ** rng.randrange(-25, 25)) for _ in range(20000)]
    texts += ["0.0", "-0.0", "1e0", "1E+5", "1e-5", "1234567890123456789", "0.30000000000000004", "9007199254740993", "4.35", "1e19",
              "5e-20", "0.5000000000000000000000000", "9.999999999999999e22", "1e22"]
    return texts


def near_halfway_texts(seed=17, count=12000):
    """Decimal texts on both sides of rounding decisions: for random doubles d in the range to_double takes, the exact midpoint
    m of d and nextafter(d, inf) printed to 17, 18 and 19 significant digits, rounded down and up, and m itself where it has
    at most 19 significant digits (every d in [2^50, 10^19) gives one: exact ties, decided to even).  Both signs."""
    import decimal
    import random
    rng = random.Random(seed)
    ds = []
    for _ in range(count):
        r = rng.random()
        if r < 0.5:       # any magnitude the 19-digit long division reaches
            d = rng.uniform(1.0, 10.0) * 10.0 ** rng.randrange(-3, 38)
        elif r < 0.8:     # integers above 2^53: the midpoint is an odd integer or ends in .5 / .25 / .125
            d = float(rng.randrange(2 ** 50, 10 ** 19))
        else:             # the Clinger range: short mantissas, |exponent| <= 22
            d = rng.uniform(1.0, 10.0) * 10.0 ** rng.randrange(-22, 16)
        ds.append(d)
    texts = []
    with decimal.localcontext() as ctx:
        ctx.prec = 1000
        for d in ds:
            mid = (decimal.Decimal(d) + decimal.Decimal(math.nextafter(d, math.inf))) / 2
            sign = "-" if rng.random() < 0.2 else ""
            if len(mid.normalize().as_tuple().digits) <= 19:
                texts.append(sign + str(mid.normalize()))
            for prec in (17, 18, 19):
                for rounding in (decimal.ROUND_FLOOR, decimal.ROUND_CEILING):
                    c = decimal.Context(prec=prec, rounding=rounding)
                    texts.append(sign + str(c.plus(mid)))
    return texts


def boundary_texts():
    """(texts, must_decline): powers of ten 1e-22 .. 1e19 in several spellings, mantissas at 2^53 and 2^53 + 1, 19- and
    20-significant-digit texts (the latter declined), leading-zero fractions, signed zeros."""
    texts, decline = [], []
    for k in range(-22, 20):
        texts += ["1e%d" % k, "1E%+d" % k, "10e%d" % (k - 1), "%se%d" % ("1" + "0" * 5, k - 5)]
        if k < 0:
            texts.append("0." + "0" * (-k - 1) + "1")
        else:
            texts.append("1" + "0" * k)
    for w in (2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, 2 ** 54 - 1, 2 ** 54 + 1, 10 ** 19 - 1):
        for e in (-22, -20, -19, -18, -10, -1, 0, 1, 5, 19):
            texts.append("%de%d" % (w, e))
    nineteen = ["1234567890123456789", "9999999999999999999", "1000000000000000001", "9223372036854775807", "9223372036854775808",
                "18446744073709551615"[:19]]
    for m in nineteen:
        texts += [m, m[:1] + "." + m[1:], "0." + m, m + "e19", m + "e-19", m[:10] + "." + m[10:] + "e-5", m + "0", m + ".000"]
        decline += [m + "1", m[:1] + "." + m[1:] + "7", "0." + m + "3", m + "5e-3", m[:12] + "." + m[12:] + "9"]
    texts += ["0." + "0" * 21 + "1", "0." + "0" * 21 + "12345", "0.0000000000000000000001", "-0.0000000000000000000001", "-0", "-0.0",
              "0e5", "0E-5", "-0e0", "0.000", "0.5", "-1.5e-22", "9.999999999999999999", "1.0000000000000000000"]
    decline += ["0." + "0" * 22 + "1", "1e20", "1e-23", "12345678901234567891", "1.2345678901234567891"]
    return texts, decline


def repr_doubles():
    """float64 values for float.__repr__: random in every range, random bit patterns, every power of two and of ten,
    subnormals, the extremes, inf and NaN."""
    rng = np.random.default_rng(1)
    bits = rng.integers(0, 2 ** 63, 40000, dtype=np.uint64).view(np.float64)
    xs = np.concatenate([rng.random(40000) * 1e4 + 1, np.floor(rng.random(20000) * 1e6), bits[np.isfinite(bits)], -bits[:500],
                         rng.random(40000) * 10.0 ** rng.integers(-30, 30, 40000), np.round(rng.random(20000), 5),
                         [2.0 ** k for k in range(-1074, 1024)], [10.0 ** k for k in range(-323, 309)],
                         [0.0, -0.0, 1.0, 1e16, 1e15, 123456789012345680.0, 1e-5, 1e-4, 5e-324, 1.7976931348623157e308,
                          2.2250738585072014e-308, 1e22, 1e23, float("inf"), float("-inf"), float("nan")]])
    return np.ascontiguousarray(xs)


def pack_number_texts(texts):
    """texts -> (blob uint8, off int64 [len + 1]) for kc_debug_parse_doubles(_device)."""
    enc = [t.encode() for t in texts]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in enc], out=off[1:])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8).copy()
    return blob, off


def cpython_doubles(texts):
    """float(t) for every JSON number text (CPython's correctly rounded conversion), as a float64 array.  This is
    float(json.loads(t)) except for "-0", which json.loads reads as the int 0: to_double keeps the sign, and the JSON paths
    carry the int-ness of the text apart from the value."""
    assert all(isinstance(json.loads(t), (int, float)) for t in texts)
    return np.array([float(t) for t in texts], dtype=np.float64)


# ----------------------------------------------------------------------------- mutated candidate texts

MUTATE_ALPHABET = '{}[]",:0123456789.eE-+ntf \n\t\\u00e9abcxyzNI'


def mutate(rng, text):
    """One or two random character substitutions, deletions or insertions (JSON punctuation, digits, escapes, letters)."""
    chars = list(text)
    for _ in range(rng.randrange(1, 3)):
        i, r = rng.randrange(len(chars)), rng.random()
        if r < 0.4:
            chars[i] = rng.choice(MUTATE_ALPHABET)
        elif r < 0.7:
            del chars[i]
        else:
            chars.insert(i, rng.choice(MUTATE_ALPHABET))
    return "".join(chars)


def general_and_mutated_records(seed=11):
    """{n: records}: general flat records with phrases, big ints and missing keys, nested records, and flat records with about
    half their candidate texts mutated (most of those are invalid JSON or change a value's type)."""
    import random
    from tests.test_gpu_json import _random_nested_record, _random_record
    from tests.test_jsongpu_host_logic import _flat_record
    rng = random.Random(seed)
    by_n = {}
    for _ in range(600):
        n = rng.choice([2, 3, 5, 8, 16])
        by_n.setdefault(n, []).append(_random_record(rng, n))
    for _ in range(200):
        n = rng.choice([2, 3, 5])
        by_n.setdefault(n, []).append(_random_nested_record(rng, n))
    for _ in range(800):
        n = rng.choice([2, 3, 5])
        texts = [mutate(rng, t) if rng.random() < 0.5 else t for t in _flat_record(rng, n)]
        if all(texts):
            by_n.setdefault(n, []).append(texts)
    return by_n


def oracle_run(plan):
    """Stand-in for Plan.run(): evaluate the recorded groups with the columnar C ORACLE instead of the GPU.
    Used by CPU tests of the host prologue/epilogue only."""
    from oracle import columnar as OC
    out = {}
    if plan.vote_rows:
        _, meta = OC.vote(np.asarray(plan.vote_rows, dtype=np.int32), None)
        out["vote_meta"] = meta
    if plan.num_rows:
        value, meta = OC.numeric(np.asarray(plan.num_rows, dtype=np.float64), plan.rel_eps, plan.abs_eps)
        out["num_value"], out["num_meta"] = value, meta
    if plan.medoid_groups:
        out["medoid_idx"], out["medoid_avg"] = OC.medoid(plan.medoid_groups)
    return out


def _fnv1a(strings_u8):
    """32-bit FNV-1a of each row of a uint8 [S, L] array (K4's duplicate filter, kc_medoid.cuh)."""
    h = np.full(len(strings_u8), 2166136261, dtype=np.uint32)
    for q in range(strings_u8.shape[1]):
        h = (h ^ strings_u8[:, q]) * np.uint32(16777619)
    return h


def _fnv_collision(seed=1):
    """Two different [a-z0-9] strings of length 8 with the same 32-bit FNV-1a hash, by a birthday search."""
    rng = np.random.default_rng(seed)
    alphabet = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789", dtype=np.uint8)
    strs = np.zeros((0, 8), dtype=np.uint8)
    while True:
        strs = np.concatenate([strs, alphabet[rng.integers(0, 36, (50000, 8))]])
        h = _fnv1a(strs)
        order = np.argsort(h, kind="stable")
        same = np.nonzero(h[order][1:] == h[order][:-1])[0]
        for s in same:
            a, b = strs[order[s]].tobytes().decode(), strs[order[s + 1]].tobytes().decode()
            if a != b:
                return a, b


_WORDS = ("invoice total due amount net gross payment bank transfer within thirty days from receipt of goods and services "
          "the a an of to acme corp ltd gmbh street road avenue suite floor new york london paris berlin 2024 2025 q1 q2 "
          "ref no id number 000123 77 ab-12 x y z").split()


def random_string_groups(rng, n_groups, max_k=16, long_frac=0.1):
    """Groups of 2..max_k multi-word strings: noisy copies of a base phrase (the shape of LLM string fields)."""
    groups = []
    for _ in range(n_groups):
        k = int(rng.integers(2, max_k + 1))
        base = [_WORDS[int(i)] for i in rng.integers(0, len(_WORDS), int(rng.integers(3, 9)))]
        grp = []
        for _c in range(k):
            words = list(base)
            r = rng.random()
            if r < 0.35:
                pass
            elif r < 0.6:
                words[int(rng.integers(0, len(words)))] = _WORDS[int(rng.integers(0, len(_WORDS)))]
            elif r < 0.75:
                words = words[: max(1, len(words) - int(rng.integers(1, 3)))]
            elif r < 0.9:
                words = words + [_WORDS[int(i)] for i in rng.integers(0, len(_WORDS), int(rng.integers(1, 4)))]
            else:
                words = [w.upper() if rng.random() < 0.5 else w + "," for w in words]
            s = " ".join(words)
            if rng.random() < 0.03:
                s = ""
            grp.append(s)
        if rng.random() < long_frac:  # one long member is still inside K4's contract (pattern = the shorter string)
            grp[int(rng.integers(0, k))] = " ".join(_WORDS[int(i)] for i in rng.integers(0, len(_WORDS), 40))
        groups.append(grp)
    return groups


def consolidate_json_with_oracle(records):
    """kc_json_plan -> the C ORACLE in the place of K1 / K2 / K4 -> kc_json_emit: the host logic of the native JSON path
    (H1) checked on a machine without a GPU.  Same return convention as _native.consolidate_json."""
    import ctypes as c
    from k_llms_b200 import _native as K
    from oracle import columnar as OC
    lib = K.load()
    R = len(records)
    if R == 0:
        return []
    n = len(records[0])
    assert all(len(r) == n for r in records)
    blobs = [t.encode("utf-8") for r in records for t in r]
    texts = (c.c_char_p * (R * n))(*blobs)
    lens = (c.c_int64 * (R * n))(*[len(b) for b in blobs])
    h = c.c_void_p()
    K.check(lib.kc_json_plan(c.cast(texts, c.c_void_p), c.cast(lens, c.c_void_p), R, n, 4, c.byref(h)))
    try:
        vc, nc, mc, so, go = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        gv, gx, gm, mx = c.c_int64(), c.c_int64(), c.c_int64(), c.c_int32()
        K.check(lib.kc_json_inputs(h, c.byref(vc), c.byref(gv), c.byref(nc), c.byref(gx), c.byref(mc), c.byref(so), c.byref(go),
                                   c.byref(gm), c.byref(mx)))
        vmeta = np.zeros(max(gv.value, 1), dtype=np.uint32)
        nvalue, nmeta = np.zeros(max(gx.value, 1), dtype=np.float64), np.zeros(max(gx.value, 1), dtype=np.uint32)
        midx, mavg = np.zeros(max(gm.value, 1), dtype=np.int32), np.zeros(max(gm.value, 1), dtype=np.float64)
        if gv.value:
            codes = np.ctypeslib.as_array(c.cast(vc, c.POINTER(c.c_int8)), shape=(gv.value, n)).astype(np.int32)
            _, vmeta = OC.vote(codes, None)
        if gx.value:
            vals = np.ctypeslib.as_array(c.cast(nc, c.POINTER(c.c_double)), shape=(gx.value, n)).copy()
            nvalue, nmeta = OC.numeric(vals)
        if gm.value:
            OC.lib().ko_medoid_str(mc, so, go, gm.value, midx.ctypes.data, mavg.ctypes.data)
        out_c, out_l, status = (c.c_void_p * R)(), (c.c_void_p * R)(), (c.c_uint8 * R)()
        K.check(lib.kc_json_emit(h, vmeta.ctypes.data, nvalue.ctypes.data, nmeta.ctypes.data, midx.ctypes.data, mavg.ctypes.data,
                                 c.cast(out_c, c.c_void_p), c.cast(out_l, c.c_void_p), c.cast(status, c.c_void_p)))
        res = [(c.string_at(out_c[i]).decode("ascii"), c.string_at(out_l[i]).decode("ascii")) if status[i] == 0 else None for i in range(R)]
        lib.kc_free_strings(c.cast(out_c, c.c_void_p), R)
        lib.kc_free_strings(c.cast(out_l, c.c_void_p), R)
        return res
    finally:
        lib.kc_json_free(h)


def jsongpu_with_oracle(records, seq=None, flags=0):
    """The DEVICE JSON path's phases (kc_jsongpu.cuh) instantiated on the host: kc_debug_jsongpu_plan_flags -> the oracles in the
    kernels' places -> kc_debug_jsongpu_emit_weighted.  K1: the C oracle's vote, or with seq (float32 [R*n] candidate sums) its
    likelihood-weighted vote over the group records (K3b); K2: the C oracle, or with JSON_NUMERIC_MEDOID in flags numpy's medoid
    (K5, tests.async_native_oracle.numeric_medoid); K4: the C oracle.  Returns (pairs, status): pairs[r] = (content,
    likelihoods) or None where the device path declines the record (status[r] = its reason code)."""
    import ctypes as c
    from k_llms_b200 import _native as K
    from oracle import columnar as OC
    from tests.async_native_oracle import numeric_medoid
    lib = K.load()
    R = len(records)
    if R == 0:
        return [], []
    blob, off, n = K.pack_texts(records, pinned=False)
    h = c.c_void_p()
    K.check(lib.kc_debug_jsongpu_plan_flags(blob.ctypes.data, off.ctypes.data, R, n, flags, c.byref(h)))
    try:
        vc, nc, st, gr = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        gv, gx = c.c_int64(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_inputs(h, c.byref(vc), c.byref(gv), c.byref(nc), c.byref(gx), c.byref(st)))
        vmeta, vweight = np.zeros(max(gv.value, 1), dtype=np.uint32), np.zeros(max(gv.value, 1), dtype=np.float32)
        if gv.value:
            codes = np.ctypeslib.as_array(c.cast(vc, c.POINTER(c.c_int8)), shape=(gv.value, n)).astype(np.int32)
            if seq is None:
                _, vmeta = OC.vote(codes, None)
            else:
                K.check(lib.kc_debug_jsongpu_group_records(h, c.byref(gr)))
                rec = np.ctypeslib.as_array(c.cast(gr, c.POINTER(c.c_int32)), shape=(gv.value,)).copy()
                assert (rec >= 0).all() and (rec < R).all()
                _, vmeta, vweight = OC.weighted_vote(codes[:, None, :], np.asarray(seq, dtype=np.float32).reshape(R, n)[rec])
        nvalue, nmeta = np.zeros(max(gx.value, 1), dtype=np.float64), np.zeros(max(gx.value, 1), dtype=np.uint32)
        best, avg = np.zeros(max(gx.value, 1), dtype=np.int32), np.zeros(max(gx.value, 1), dtype=np.float64)
        if gx.value:
            cells = np.ctypeslib.as_array(c.cast(nc, c.POINTER(c.c_double)), shape=(gx.value, n)).copy()
            if flags & K.JSON_NUMERIC_MEDOID:
                best, avg = numeric_medoid(cells)
            else:
                nvalue, nmeta = OC.numeric(cells)
        K.check(lib.kc_debug_jsongpu_set_numeric_medoid(h, best.ctypes.data, avg.ctypes.data))
        mc, so, go, gm = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_medoid_inputs(h, c.byref(mc), c.byref(so), c.byref(go), c.byref(gm)))
        midx, mavg = np.zeros(max(gm.value, 1), dtype=np.int32), np.zeros(max(gm.value, 1), dtype=np.float64)
        if gm.value:
            OC.lib().ko_medoid_str(mc, so, go, gm.value, midx.ctypes.data, mavg.ctypes.data)
        K.check(lib.kc_debug_jsongpu_set_medoid(h, midx.ctypes.data, mavg.ctypes.data))
        pc, po, pl, plo = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        K.check(lib.kc_debug_jsongpu_emit_weighted(h, vmeta.ctypes.data, None if seq is None else vweight.ctypes.data, nvalue.ctypes.data,
                                                   nmeta.ctypes.data, c.byref(pc), c.byref(po), c.byref(pl), c.byref(plo)))
        # a record can still be declined while encoding (number range): read the statuses after emit
        status = np.ctypeslib.as_array(c.cast(st, c.POINTER(c.c_uint8)), shape=(R,)).copy()
        co = np.ctypeslib.as_array(c.cast(po, c.POINTER(c.c_int64)), shape=(R + 1,))
        lo = np.ctypeslib.as_array(c.cast(plo, c.POINTER(c.c_int64)), shape=(R + 1,))
        pairs = [None if status[r] else (c.string_at(pc.value + int(co[r]), int(co[r + 1] - co[r])).decode("ascii"),
                                         c.string_at(pl.value + int(lo[r]), int(lo[r + 1] - lo[r])).decode("ascii")) for r in range(R)]
        return pairs, [int(s) for s in status]
    finally:
        lib.kc_debug_jsongpu_free(h)


# ----------------------------------------------------------------------------- which kernels ran (torch.profiler)

def kernel_key(name):
    """'void kc::vote_tma_kernel<32, 8, 2, true>(CUtensorMap_st, ...)' -> 'vote_tma_kernel<32,8,2,true>'."""
    m = re.search(r"kc::(\w+(?:<[^()]*>)?)\(", name)
    return m.group(1).replace(" ", "") if m else None


@contextlib.contextmanager
def profiled():
    """torch.profiler over the block.  In a full-suite run the kernels launched right after the profiler started were
    missing from its record, so a few throwaway kernels go first."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        x = torch.zeros(1024, device="cuda")
        for _ in range(8):
            x.add_(1)
        torch.cuda.synchronize()
        yield prof
        torch.cuda.synchronize()


def kernels_seen(prof):
    """(the kernel keys the profiler recorded, whether it recorded any CUDA kernel at all)."""
    import torch
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {k for k in map(kernel_key, names) if k}, bool(names)


def assert_kernels_ran(prof, expected):
    import pytest
    seen, any_names = kernels_seen(prof)
    if not any_names:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable)")
    missing = sorted(set(expected) - seen)
    assert not missing, (missing, sorted(seen))
