"""Shared test helpers: golden loading, strict equality (float bits, key order), a CPU stand-in device."""
import json
import math
import os

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


def raising_embeddings(texts):
    raise RuntimeError("no network in tests")


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


def jsongpu_with_oracle(records):
    """The DEVICE JSON path's phases (kc_jsongpu.cuh) instantiated on the host: kc_debug_jsongpu_plan -> the C ORACLE in the
    place of K1 / K2 / K4 -> kc_debug_jsongpu_emit.  Returns (pairs, status): pairs[r] = (content, likelihoods) or None where the
    device path declines the record (status[r] = its reason code)."""
    import ctypes as c
    from k_llms_b200 import _native as K
    from oracle import columnar as OC
    lib = K.load()
    R = len(records)
    if R == 0:
        return [], []
    blob, off, n = K.pack_texts(records, pinned=False)
    h = c.c_void_p()
    K.check(lib.kc_debug_jsongpu_plan(blob.ctypes.data, off.ctypes.data, R, n, c.byref(h)))
    try:
        vc, nc, st = c.c_void_p(), c.c_void_p(), c.c_void_p()
        gv, gx = c.c_int64(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_inputs(h, c.byref(vc), c.byref(gv), c.byref(nc), c.byref(gx), c.byref(st)))
        status = np.ctypeslib.as_array(c.cast(st, c.POINTER(c.c_uint8)), shape=(R,)).copy()
        vmeta = np.zeros(max(gv.value, 1), dtype=np.uint32)
        nvalue, nmeta = np.zeros(max(gx.value, 1), dtype=np.float64), np.zeros(max(gx.value, 1), dtype=np.uint32)
        if gv.value:
            codes = np.ctypeslib.as_array(c.cast(vc, c.POINTER(c.c_int8)), shape=(gv.value, n)).astype(np.int32)
            _, vmeta = OC.vote(codes, None)
        if gx.value:
            vals = np.ctypeslib.as_array(c.cast(nc, c.POINTER(c.c_double)), shape=(gx.value, n)).copy()
            nvalue, nmeta = OC.numeric(vals)
        mc, so, go, gm = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_medoid_inputs(h, c.byref(mc), c.byref(so), c.byref(go), c.byref(gm)))
        midx, mavg = np.zeros(max(gm.value, 1), dtype=np.int32), np.zeros(max(gm.value, 1), dtype=np.float64)
        if gm.value:   # the C oracle in K4's place
            OC.lib().ko_medoid_str(mc, so, go, gm.value, midx.ctypes.data, mavg.ctypes.data)
        K.check(lib.kc_debug_jsongpu_set_medoid(h, midx.ctypes.data, mavg.ctypes.data))
        pc, po, pl, plo = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        K.check(lib.kc_debug_jsongpu_emit(h, vmeta.ctypes.data, nvalue.ctypes.data, nmeta.ctypes.data, c.byref(pc), c.byref(po),
                                          c.byref(pl), c.byref(plo)))
        # a record can still be declined while encoding (number range): re-read the statuses
        status = np.ctypeslib.as_array(c.cast(st, c.POINTER(c.c_uint8)), shape=(R,)).copy()
        co = np.ctypeslib.as_array(c.cast(po, c.POINTER(c.c_int64)), shape=(R + 1,))
        lo = np.ctypeslib.as_array(c.cast(plo, c.POINTER(c.c_int64)), shape=(R + 1,))
        pairs = []
        for r in range(R):
            if status[r]:
                pairs.append(None)
            else:
                pairs.append((c.string_at(pc.value + int(co[r]), int(co[r + 1] - co[r])).decode("ascii"),
                              c.string_at(pl.value + int(lo[r]), int(lo[r + 1] - lo[r])).decode("ascii")))
        return pairs, list(status)
    finally:
        lib.kc_debug_jsongpu_free(h)
