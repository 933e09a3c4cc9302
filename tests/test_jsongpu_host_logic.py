"""Logic of the DEVICE JSON path (H1g, k_llms_b200/csrc/kc_jsongpu.cuh) on a machine without a GPU: its phase functions are
__host__ __device__, and the kc_debug_jsongpu_* hooks run them on the host lane by lane with the C oracle in the place of
K1 / K2.  Everything the path accepts must be byte-identical to the reference's client order (json.loads -> align ->
consensus -> json.dumps, restated by the object-level oracle); everything else it must decline.  Also pins the exact
decimal -> float64 conversion and the shortest-digits float.__repr__ of kc_jsoncore.cuh, and round(x, 5) of kc_internal.h,
against CPython."""
import json
import random

import numpy as np

from k_llms_b200 import _native as K
from tests.helpers import (boundary_texts, cpython_doubles, jsongpu_with_oracle, near_halfway_texts, number_texts, pack_number_texts,
                           repr_doubles)
from tests.test_gpu_json import _expected, _random_nested_record, _random_record


def s32_texts(R, n, seed):
    """The bench workload as candidate texts: schema S32 (16 string-enum with case/punctuation variants, 8 bool, 6 int,
    2 float fields), p_agree 0.8, p_none 0.05."""
    from k_llms_b200 import synth
    codes, _none, vals = synth.s32_numpy(R, n, seed)
    vocab = ["alpha", "Bravo", "charlie", "DELTA", "echo", "foxtrot", "golf", "Hotel"]
    variants = [lambda w: w, lambda w: w.upper(), lambda w: w.lower() + "!", lambda w: " " + w]
    out = []
    for r in range(R):
        rec = []
        for c in range(n):
            d = {}
            for f in range(16):
                k = int(codes[r, f, c])
                d[f"f{f:02d}"] = None if k < 0 else variants[(r + c + f) % 4](vocab[k])
            for f in range(16, 24):
                k = int(codes[r, f, c])
                d[f"f{f:02d}"] = None if k < 0 else bool(k)
            for f in range(8):
                v = vals[r, f, c]
                d[f"f{24 + f:02d}"] = None if v != v else (int(v) if f < 6 else float(v))
            rec.append(json.dumps(d))
        out.append(rec)
    return out


def test_s32_records_all_on_the_device_path():
    for n in (2, 3, 5, 16, 33):
        recs = s32_texts(40 if n < 33 else 12, n, 100 + n)
        pairs, status = jsongpu_with_oracle(recs)
        assert not any(status), status
        for texts, got in zip(recs, pairs):
            assert got == _expected(texts), texts


def _flat_record(rng, n):
    """Flat records in the device path's territory, with everything that must still come out right: shuffled key order in the
    text vs sorted output, case / punctuation variants, empty strings, two-word strings, ints that print as floats, long
    floats, exponents, negative zero, bool/None mixes, single non-None numerics, strings inside numeric fields."""
    n_fields = rng.randrange(1, 9)
    names = rng.sample(["zeta", "Alpha", "b", "a", "aa", "a_b", "k1", "k10", "k2", "Z", "m-n", "id"], n_fields)
    kinds = [rng.choice(["enum", "bool", "int", "float", "sci", "tie", "one", "numstr", "allnull", "two"]) for _ in names]
    words = ["alpha", "Bravo", "charlie", "DELTA", "echo", "fox-trot", "", "a b", "Hotel!", "hotel", " HOTEL "]
    truth = {}
    for k, kind in zip(names, kinds):
        truth[k] = {"enum": lambda: rng.choice(words), "bool": lambda: rng.random() < 0.5, "int": lambda: rng.randrange(-50, 10 ** rng.randrange(1, 9)),
                    "float": lambda: rng.uniform(-1e3, 1e5), "sci": lambda: rng.choice([1e-7, 2.5e-5, 1e16, 1.5e17, 123456789.125, 0.0, -0.0, 1e-4]),
                    "tie": lambda: rng.choice([1, 2, 100, 102.9, 105.8]), "one": lambda: rng.choice([7, 7.5, -0.0, 12345678901234567]),
                    "numstr": lambda: rng.randrange(0, 100), "allnull": lambda: None, "two": lambda: rng.choice(["new york", "New  York", "los angeles"])}[kind]()
    texts = []
    for _c in range(n):
        d = {}
        for k, kind in zip(names, kinds):
            v = truth[k]
            r = rng.random()
            if kind == "one":
                v = v if _c == n // 2 else None
            elif r < 0.3:
                v = {"enum": lambda: rng.choice(words).upper(), "bool": lambda: rng.random() < 0.5, "int": lambda: rng.randrange(0, 1000),
                     "float": lambda: rng.uniform(0, 10), "sci": lambda: truth[k] * rng.choice([1.02, 0.97, 10.0, -1.0]),
                     "tie": lambda: rng.choice([1, 2, 100, 102.9, 105.8]), "numstr": lambda: rng.choice(["12", True, 3.5]),
                     "allnull": lambda: None, "two": lambda: rng.choice(["new york", "NEW YORK!", "boston"])}[kind]()
            elif r > 0.92:
                v = None
            d[k] = v
        t = json.dumps(d)
        if rng.random() < 0.1:
            t = t.replace(", ", " ,\n\t").replace("{", "{ ").replace("}", " }\r\n")
        if rng.random() < 0.05:
            t = t.replace(": ", ":")
        texts.append(t)
    return texts


def test_flat_records_match_client_order():
    rng = random.Random(3)
    by_n, on_device = {}, 0
    for _ in range(1500):
        n = rng.choice([2, 3, 4, 5, 8, 16, 20, 40])
        by_n.setdefault(n, []).append(_flat_record(rng, n))
    for _n, recs in by_n.items():
        pairs, status = jsongpu_with_oracle(recs)
        for texts, got, st in zip(recs, pairs, status):
            if got is None:
                continue
            on_device += 1
            assert got == _expected(texts), (texts, st)
    assert on_device > 1200, on_device


PHRASES = ["the quick brown fox", "The Quick Brown Fox!", "the quick brown fax", "a quick brown fox jumps", "net 30 days", "Net 30 Days.",
           "payment due on receipt", "- - -", "x y z", "invoice total due within thirty days of receipt of the goods delivered",
           "two words", "one", "", "line one\nline two", "say \"net 30\" days", "a/b c\\d e", "tab\tseparated\twords here", "x\ty", "the quick\nbrown fox"]


def _phrase_record(rng, n):
    """Flat records with multi-word string fields (similarity medoid, K4) next to voted and numeric fields: agreeing and
    disagreeing phrases, case / punctuation variants, Nones, a single non-None phrase, one long phrase (two long ones are the
    embeddings service's: declined), strings that normalise to nothing."""
    n_fields = rng.randrange(1, 6)
    names = rng.sample(["terms", "note", "a", "b", "zz", "Address"], n_fields)
    kinds = [rng.choice(["phrase", "phrase", "enum", "int", "bool"]) for _ in names]
    truth = {k: {"phrase": lambda: rng.choice(PHRASES[:10]), "enum": lambda: rng.choice(["alpha", "Bravo", "two words"]),
                 "int": lambda: rng.randrange(0, 1000), "bool": lambda: rng.random() < 0.5}[kind]() for k, kind in zip(names, kinds)}
    lone = rng.random() < 0.1
    texts = []
    for c in range(n):
        d = {}
        for k, kind in zip(names, kinds):
            v, r = truth[k], rng.random()
            if kind == "phrase" and lone:
                v = v if c == n - 1 else None
            elif r < 0.35:
                v = {"phrase": lambda: rng.choice(PHRASES), "enum": lambda: rng.choice(["ALPHA", "bravo!", "x"]),
                     "int": lambda: rng.randrange(0, 1000), "bool": lambda: rng.random() < 0.5}[kind]()
            elif r > 0.9:
                v = None
            d[k] = v
        texts.append(json.dumps(d))
    return texts


def test_phrase_fields_take_the_medoid():
    rng = random.Random(29)
    by_n, on_device, with_groups = {}, 0, 0
    for _ in range(1500):
        n = rng.choice([2, 3, 4, 5, 8, 16, 33])
        by_n.setdefault(n, []).append(_phrase_record(rng, n))
    for _n, recs in by_n.items():
        pairs, status = jsongpu_with_oracle(recs)
        for texts, got, st in zip(recs, pairs, status):
            if got is None:
                continue
            on_device += 1
            with_groups += any(len(v.split()) >= 3 for t in texts for v in json.loads(t).values() if isinstance(v, str))
            assert got == _expected(texts), (texts, st)
    assert on_device > 1200 and with_groups > 700, (on_device, with_groups)


def test_two_character_escapes_in_values():
    """Escapes stay in the token: skipped by the sanitiser (\\n must not leave an 'n'), one character each for the 50-character
    rule, whitespace for the word count where Python's split() says so, printed as json.dumps prints them (\\/ -> /)."""
    esc = ['\\"', '\\\\', '\\/', '\\b', '\\f', '\\n', '\\r', '\\t']
    rng = random.Random(5)
    recs = []
    for _ in range(400):
        n = rng.choice([2, 3, 5, 8])
        base = [rng.choice(["alpha", "n", "t", "big cat", "Net", "x", ""]) for _ in range(rng.randrange(1, 5))]
        texts = []
        for _c in range(n):
            parts = list(base)
            if rng.random() < 0.3:
                parts[rng.randrange(len(parts))] = rng.choice(["ALPHA", "n!", "dog"])
            joined = "".join(p + rng.choice(esc + [" ", " ", "-"]) for p in parts) + rng.choice(["", "end", "\\n"])
            texts.append('{"k": "%s", "m": %s}' % (joined, rng.choice(["1", "null", '"a\\tb"'])))
        recs.append(texts)
    edge = [['{"k": "%s"}' % ("ab\\n" * 17 + " x y"), '{"k": "%s"}' % ("ab\\n" * 16 + " x y")],    # 55 and 52 characters: both long
            ['{"k": "%s"}' % ("ab\\n" * 16 + "x y"), '{"k": "%s"}' % ("ab\\n" * 15 + " x y z")[:-1]]]   # 51 and 50 characters: one long
    pairs, status = jsongpu_with_oracle(edge)
    assert status[0] != 0 and status[1] == 0 and pairs[1] == _expected(edge[1])
    accepted = 0
    for n in (2, 3, 5, 8):
        group = [r for r in recs if len(r) == n]
        pairs, status = jsongpu_with_oracle(group)
        for texts, got in zip(group, pairs):
            if got is not None:
                accepted += 1
                assert got == _expected(texts), texts
    assert accepted > 200, accepted


def _shaped_record(rng, n):
    """n candidates of ONE shape (same keys in the same textual order at every level, keys not in sorted order) whose leaves
    disagree: nested objects up to depth 4 next to every kind of scalar field."""
    def shape(depth):
        keys = rng.sample(["zeta", "Alpha", "b", "a", "aa", "k1", "k10", "k2", "Z", "id", "name", "addr"], rng.randrange(1, 6))
        out = []
        for k in keys:
            if depth < 4 and rng.random() < 0.3:
                out.append((k, shape(depth + 1)))
            else:
                out.append((k, rng.choice(["enum", "bool", "int", "float", "phrase", "allnull", "one"])))
        return out

    def truth_of(sh):
        return [(k, truth_of(v) if isinstance(v, list) else
                 {"enum": lambda: rng.choice(["alpha", "Bravo", "two words", ""]), "bool": lambda: rng.random() < 0.5,
                  "int": lambda: rng.randrange(-5, 10 ** rng.randrange(1, 7)), "float": lambda: rng.uniform(-10, 1e4),
                  "phrase": lambda: rng.choice(PHRASES[:10]), "allnull": lambda: None, "one": lambda: rng.choice([7, "solo", 2.5])}[v]())
                for k, v in sh]

    def candidate(sh, tr, c):
        d = {}
        for (k, kind), (_k, tv) in zip(sh, tr):
            if isinstance(kind, list):
                d[k] = candidate(kind, tv, c)
                continue
            v, r = tv, rng.random()
            if kind == "one":
                v = v if c == 0 else None
            elif r < 0.3:
                v = {"enum": lambda: rng.choice(["ALPHA", "bravo!", "x"]), "bool": lambda: rng.random() < 0.5, "int": lambda: rng.randrange(0, 100),
                     "float": lambda: rng.uniform(0, 10), "phrase": lambda: rng.choice(PHRASES), "allnull": lambda: None}[kind]()
            elif r > 0.92:
                v = None
            d[k] = v
        return d

    sh = shape(1)
    tr = truth_of(sh)
    texts = []
    for c in range(n):
        t = json.dumps(candidate(sh, tr, c))
        if rng.random() < 0.1:
            t = t.replace(", ", " ,\n\t").replace("{", "{ ").replace("}", " }\r\n")
        texts.append(t)
    return texts


def test_nested_objects_of_one_shape():
    rng = random.Random(41)
    by_n, on_device, nested = {}, 0, 0
    for _ in range(1500):
        n = rng.choice([2, 3, 4, 5, 8, 16, 33])
        by_n.setdefault(n, []).append(_shaped_record(rng, n))
    for _n, recs in by_n.items():
        pairs, status = jsongpu_with_oracle(recs)
        for texts, got, st in zip(recs, pairs, status):
            if got is None:
                continue
            on_device += 1
            nested += any(isinstance(v, dict) for v in json.loads(texts[0]).values())
            assert got == _expected(texts), (texts, st)
    assert on_device > 1300 and nested > 700, (on_device, nested)


def test_general_records_accepted_or_declined():
    """The generators of the host-path tests (missing keys, nested objects, phrases, big ints, escapes, mixed types): the device
    path declines most of them; what it accepts must be exact."""
    rng = random.Random(11)
    by_n = {}
    for _ in range(600):
        n = rng.choice([2, 3, 5, 8, 16])
        by_n.setdefault(n, []).append(_random_record(rng, n))
    for _ in range(200):
        n = rng.choice([2, 3, 5])
        by_n.setdefault(n, []).append(_random_nested_record(rng, n))
    accepted = declined = 0
    for _n, recs in by_n.items():
        pairs, _status = jsongpu_with_oracle(recs)
        for texts, got in zip(recs, pairs):
            if got is None:
                declined += 1
                continue
            accepted += 1
            assert got == _expected(texts), texts
    assert accepted > 50 and declined > 50, (accepted, declined)


def test_mutated_texts_accepted_or_declined():
    """Random byte edits (broken JSON, stray tokens, escapes, non-ASCII bytes): never a wrong answer."""
    rng = random.Random(7)
    alphabet = '{}[]",:0123456789.eE-+ntf \n\t\\u00e9\xe9abcxyzNI'

    def mutate(text):
        chars = list(text)
        for _ in range(rng.randrange(1, 3)):
            i, r = rng.randrange(len(chars)), rng.random()
            if r < 0.4:
                chars[i] = rng.choice(alphabet)
            elif r < 0.7:
                del chars[i]
            else:
                chars.insert(i, rng.choice(alphabet))
        return "".join(chars)

    by_n, accepted = {}, 0
    for _ in range(1200):
        n = rng.choice([2, 3, 5])
        texts = [mutate(t) if rng.random() < 0.5 else t for t in _flat_record(rng, n)]
        if all(texts):
            by_n.setdefault(n, []).append(texts)
    for _n, recs in by_n.items():
        pairs, _status = jsongpu_with_oracle(recs)
        for texts, got in zip(recs, pairs):
            if got is not None:
                accepted += 1
                assert got == _expected(texts), texts
    assert accepted > 150, accepted


def test_declines_what_it_does_not_model():
    cases = {
        "unicode escape": ['{"a": "x\\u0041y"}', '{"a": "x"}'],
        "escape in a key": ['{"a\\n": "x"}', '{"a\\n": "x"}'],
        "DEL in a key": ['{"a\x7f": "x"}', '{"a\x7f": "x"}'],   # json.dumps prints DEL as \u007f: the emit prints a key's bytes
        "DEL in a value": ['{"a": "x\x7fy"}', '{"a": "x"}'],  # and without KC_JSON_UNICODE a value's
        "bad escape": ['{"a": "x\\qy"}', '{"a": "x"}'],
        "non-ascii": ['{"a": "café"}', '{"a": "cafe"}'],
        "nested here, None there": ['{"a": {"b": 1}}', '{"a": null}'],
        "nested here, scalar there": ['{"a": {"b": 1}}', '{"a": 3}'],
        "nested keys differ": ['{"a": {"b": 1}}', '{"a": {"c": 1}}'],
        "nested shapes differ": ['{"a": {"b": 1}, "c": 2}', '{"a": {"b": 1, "c": 2}}'],
        "empty nested object": ['{"a": {}}', '{"a": {}}'],
        "nested duplicate key": ['{"a": {"b": 1, "b": 2}}', '{"a": {"b": 1, "b": 2}}'],
        "nested special key": ['{"a": {"reasoning___b": "x", "c": 1}}', '{"a": {"reasoning___b": "y", "c": 1}}'],
        "list in a nested object": ['{"a": {"b": [1]}}', '{"a": {"b": [1]}}'],
        "nine levels": ['{"a": ' * 10 + '1' + '}' * 10] * 2,
        "list": ['{"a": [1, 2]}', '{"a": [1, 2]}'],
        "keys differ": ['{"a": 1, "b": 2}', '{"a": 1}'],
        "key order differs": ['{"a": 1, "b": 2}', '{"b": 2, "a": 1}'],
        "duplicate key": ['{"a": 1, "a": 2}', '{"a": 1, "a": 2}'],
        "free text": ["hello there", "hello there"],
        "top-level list": ["[1, 2]", "[1, 2]"],
        "nan": ['{"a": NaN}', '{"a": 1}'],
        "two long phrases": ['{"a": "%s"}' % ("the big cat " * 5), '{"a": "%s"}' % ("the big dog " * 5)],   # embeddings pair (cu:813)
        "phrase and number": ['{"a": "the big cat"}', '{"a": 3}'],
        "mixed str": ['{"a": "x"}', '{"a": 3}'],
        "text wrapper": ['{"text": "x"}', '{"text": "x"}'],
        "reasoning key": ['{"reasoning___a": "x", "b": 1}', '{"reasoning___a": "y", "b": 1}'],
        "empty object": ["{}", "{}"],
        "20 digits": ['{"a": 123456789012345678901}', '{"a": 1}'],
        "trailing junk": ['{"a": 1} x', '{"a": 1}'],
        "empty content": ['{"a": 1}', ''],
    }
    pairs, status = jsongpu_with_oracle(list(cases.values()))
    for (name, _), got, st in zip(cases.items(), pairs, status):
        assert got is None and st != 0, name


def parse_doubles(texts, device=None):
    """kc_debug_parse_doubles (device None: the host instantiation) or kc_debug_parse_doubles_device -> (values, ok flags)."""
    lib = K.load()
    blob, off = pack_number_texts(texts)
    out, ok = np.zeros(len(texts)), np.zeros(len(texts), dtype=np.uint8)
    if device is None:
        K.check(lib.kc_debug_parse_doubles(blob.ctypes.data, off.ctypes.data, len(texts), out.ctypes.data, ok.ctypes.data))
    else:
        K.check(lib.kc_debug_parse_doubles_device(blob.ctypes.data, off.ctypes.data, len(texts), out.ctypes.data, ok.ctypes.data, device))
    return out, ok


def assert_parsed_like_cpython(texts, out, ok):
    """Every accepted text parsed to the bits of float(json.loads(text))."""
    exp = cpython_doubles(texts)
    bad = np.nonzero(ok.astype(bool) & (out.view(np.uint64) != exp.view(np.uint64)))[0]
    assert len(bad) == 0, [(texts[i], out[i], exp[i]) for i in bad[:10]]


def test_exact_number_conversions_match_cpython():
    lib = K.load()
    texts = number_texts()
    out, ok = parse_doubles(texts)
    assert ok.sum() > 0.8 * len(texts)
    assert_parsed_like_cpython(texts, out, ok)
    # both sides of rounding decisions (exact ties, the long division's sticky bit) and the edges of the accepted range
    texts = near_halfway_texts()
    out, ok = parse_doubles(texts)
    assert ok.sum() > 0.8 * len(texts)
    assert_parsed_like_cpython(texts, out, ok)
    texts, decline = boundary_texts()
    out, ok = parse_doubles(texts + decline)
    assert not ok[len(texts):].any(), [t for t, k in zip(decline, ok[len(texts):]) if k]
    assert_parsed_like_cpython(texts + decline, out, ok)

    xs = repr_doubles()
    buf, lens = np.zeros((len(xs), 32), dtype=np.uint8), np.zeros(len(xs), dtype=np.int32)
    K.check(lib.kc_debug_float_reprs(xs.ctypes.data, len(xs), buf.ctypes.data, lens.ctypes.data))
    for i, x in enumerate(xs):
        assert bytes(buf[i, :lens[i]]).decode() == json.dumps(float(x)), repr(float(x))

    # and the products of tests/test_gpu_kernels.py::test_round5_random_products: pvf * support / present, near-half cases first
    rng = random.Random(5)
    prng = np.random.default_rng(3)
    present = prng.integers(1, 65, 200000)
    support = np.minimum((prng.random(200000) * present).astype(np.int64) + 1, present)
    pvf = prng.random(200000)
    pvf[:1000] = np.round(pvf[:1000], 5) + 5e-6
    cs = np.concatenate([[rng.random() for _ in range(50000)], [k / n for n in range(1, 65) for k in range(n + 1)],
                         pvf * (support / present)])
    out = np.zeros(len(cs))
    K.check(lib.kc_debug_round5(cs.ctypes.data, len(cs), out.ctypes.data))
    assert all(round(float(x), 5) == o for x, o in zip(cs, out))


def test_generated_s32_texts_are_json_dumps_output():
    blob, off = K.s32_texts_packed(300, 5, 9, pinned=False)  # the bench's input generator
    text = blob.tobytes()
    for i in range(0, 1500, 7):
        t = text[off[i]:off[i + 1]].decode()
        assert json.dumps(json.loads(t)) == t
