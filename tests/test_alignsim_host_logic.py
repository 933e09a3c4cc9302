"""The element-similarity pass of the batched alignment pre-pass (kc_alignsim.cuh) instantiated on the host: bit for bit
the host's generic_similarity on every pair it models, NaN on every pair it leaves to the host, and kc_align_json_batch
with that pass equal to kc_align_json record by record.  CPU only."""
import ctypes
import json
import math
import random
import struct

import pytest

from tests.helpers import load_golden
from tests.alignsim_cases import edge_pairs, element_pool, random_records

SKIP = ("reasoning___", "source___")


def _norm(s):
    return "".join(c for c in s.lower() if c.isascii() and c.isalnum())


def _falsy(v):
    return not v


def _scalar(v):
    return v is None or isinstance(v, (bool, int, float, str))


def _flat_dict(v):
    return isinstance(v, dict) and all(_scalar(x) for k, x in v.items() if not k.startswith(SKIP))


def _models_value(a, b):
    if _falsy(a) and _falsy(b):
        return True
    if a is None or b is None:
        return True
    if isinstance(a, str) and isinstance(b, str):
        if len(a) > 50 and len(b) > 50:
            return False
        if a == b:
            return True
        la, lb = len(_norm(a)), len(_norm(b))
        return max(la, lb) == 0 or min(la, lb) <= 64
    num = (bool, int, float)
    return isinstance(a, num) and isinstance(b, num) and not isinstance(a, str) and not isinstance(b, str)


def models(a, b):
    """Whether the pass decides generic_similarity(a, b) (kc_alignsim.cuh's list of what it models)."""
    if isinstance(a, dict) and isinstance(b, dict) and not (_falsy(a) and _falsy(b)):
        if not (_flat_dict(a) and _flat_dict(b)):
            return False
        keys = {k for k in list(a) + list(b) if not k.startswith(SKIP)}
        return all(_models_value(a.get(k), b.get(k)) for k in keys)
    if isinstance(a, (dict, list)) or isinstance(b, (dict, list)):
        return (_falsy(a) and _falsy(b)) or a is None or b is None
    return _models_value(a, b)


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _pass_matrix(lib, texts):
    T = len(texts)
    arr = (ctypes.c_char_p * T)(*texts)
    out = (ctypes.c_double * (T * T))()
    rc = lib.kc_debug_alignsim(ctypes.cast(arr, ctypes.c_void_p), T, ctypes.cast(out, ctypes.c_void_p))
    assert rc >= 0
    return rc, out


def test_pass_equals_host_similarity_bit_for_bit():
    from k_llms_b200 import _native as K
    lib = K.load()
    rng = random.Random(11)
    pool = element_pool(rng)
    seen = {"modelled": 0, "nan": 0}
    kinds = set()
    for it in range(60):
        T = rng.randrange(2, 80) if it else len(pool)
        elems = pool if not it else [rng.choice(pool) for _ in range(T)]
        T = len(elems)
        texts = [json.dumps(e).encode() for e in elems]
        decided, m = _pass_matrix(lib, texts)
        count = 0
        for i in range(T):
            assert math.isnan(m[i * T + i])
            for j in range(i + 1, T):
                a, b = elems[i], elems[j]
                got = m[i * T + j]
                assert _bits(got) == _bits(m[j * T + i])
                if not models(a, b):
                    assert math.isnan(got), (a, b, got)
                    seen["nan"] += 1
                    continue
                exp = ctypes.c_double()
                rc = lib.kc_debug_similarity_json(texts[i], texts[j], ctypes.byref(exp))
                assert rc == 0 and _bits(got) == _bits(exp.value), (a, b, got, exp.value)
                seen["modelled"] += 1
                count += 1
                kinds.add((type(a).__name__, type(b).__name__))
        assert decided == count
    assert seen["modelled"] > 20000 and seen["nan"] > 1000, seen
    for pair in [("int", "float"), ("bool", "int"), ("bool", "float"), ("str", "str"), ("dict", "dict"), ("NoneType", "str")]:
        assert pair in kinds or pair[::-1] in kinds, pair


def test_pass_edges():
    """The boundaries the pass models, one by one: isclose at 1 % and one ulp past, big ints, 50 / 51 raw characters,
    64 / 65 normalised characters, empty normalised forms, falsy values, dict keys."""
    from k_llms_b200 import _native as K
    lib = K.load()
    for a, b in edge_pairs():
        texts = [json.dumps(a).encode(), json.dumps(b).encode()]
        _, m = _pass_matrix(lib, texts)
        if not models(a, b):
            assert math.isnan(m[1]), (a, b, m[1])
            continue
        exp = ctypes.c_double()
        assert lib.kc_debug_similarity_json(texts[0], texts[1], ctypes.byref(exp)) == 0
        assert _bits(m[1]) == _bits(exp.value) and _bits(m[2]) == _bits(exp.value), (a, b, m[1], exp.value)


def _check_batch(records, min_support_ratio=0.51):
    from k_llms_b200 import _native as K
    counts = {}
    got = K.align_json_batch(records, min_support_ratio, device=-1, counts=counts)
    assert len(got) == len(records)
    for values, g in zip(records, got):
        exp = K.align_json(values, min_support_ratio)
        assert (g is None) == (exp is None), values
        if exp is not None:
            assert json.dumps(g) == json.dumps(exp), values
    return got, counts


def test_batch_equals_per_record_on_goldens():
    cases = load_golden("alignment")
    assert len(cases) >= 127
    got, counts = _check_batch([json.loads(json.dumps(c["values"])) for c in cases])
    assert all(g is not None for g in got)
    assert counts["device_pairs"] > 0


def test_batch_equals_per_record_on_random_structures():
    rng = random.Random(2027)
    records = random_records(rng, 5200)
    got, counts = _check_batch(records)
    assert sum(g is None for g in got) > 0 and sum(g is not None for g in got) > 4000
    assert counts["device_pairs"] > 0 and counts["host_pairs"] > 0  # nodes of > 512 elements and lists in lists: host pairs


def test_batch_other_support_ratio_and_bad_input():
    from k_llms_b200 import _native as K
    rng = random.Random(5)
    _check_batch(random_records(rng, 300), 0.3)
    assert K.align_json_batch([], 0.51, device=-1) == []
    assert K.align_json_batch([[]], 0.51, device=-1) == [None]
    lib = K.load()
    texts = (ctypes.c_char_p * 2)(b"[1, 2]", b"[1,")
    out = (ctypes.c_void_p * 2)()
    status = (ctypes.c_int32 * 1)()
    assert lib.kc_align_json_batch(ctypes.cast(texts, ctypes.c_void_p), None, 1, 2, 0.51, -1, 1, ctypes.cast(out, ctypes.c_void_p),
                                   ctypes.cast(status, ctypes.c_void_p), None) == 0
    assert status[0] == K.KC_EINVAL and not out[0] and not out[1]
    assert lib.kc_debug_alignsim(ctypes.cast(texts, ctypes.c_void_p), 1, ctypes.cast(out, ctypes.c_void_p)) == K.KC_EINVAL
    with pytest.raises(K.NativeError):
        K.check(lib.kc_align_json_batch(None, None, 1, 2, 0.51, -1, 1, None, None, None))
