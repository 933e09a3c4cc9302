"""Inputs for the tests of the batched alignment pre-pass (kc_align_json_batch, kc_alignsim.cuh): list elements that reach
every rule of the similarity pass, and candidate records with list fields of every shape the alignment meets."""
import json
import math

from oracle.gen_golden import _record_candidates, random_list_records

_WORDS = ["alpha", "Bravo", "charlie delta", "x", "", "The Quick brown fox", "the quick brown fax", "12 apples", "N/A", "!!!", "a-b c"]


def element_pool(rng):
    """List elements: scalars of every type, isclose edges, big ints, strings around the 50-raw and 64-normalised limits,
    flat and nested dicts, lists."""
    pool = [None, True, False, 0, 1, 2, -5, 99, 100, 101, 256, 1000, 10 ** 20, 10 ** 20 + 1, -(10 ** 19), 2 ** 63, 2 ** 63 - 1,
            0.0, -0.0, 1.0, 1.005, 1.01, 2.5, 100.9, 101.0, 1e-9, 3.14159, 1e300, -1e300, 7e-310]
    for base in (1.0, 100.0, 3.7, -2.5):
        edge = base + abs(base) * 0.01
        pool += [edge, math.nextafter(edge, math.inf), math.nextafter(edge, -math.inf)]
    pool += _WORDS
    pool += ["a" * 50, "b" * 50, "a" * 51, "b" * 51, "c" * 51 + "!", "ab" * 32, "ba" * 32, "ab" * 32 + "x", "q" * 65, "q" * 64 + "!!",
             "Word " * 12, "word " * 13, "x" * 40 + "?" * 30]
    pool += [{}, {"a": 1}, {"a": 1, "b": "x"}, {"c": 2, "d": "y"}, {"b": "x", "c": 2}, {"a": 1.0, "b": "X"}, {"a": True},
             {"a": None}, {"b": None}, {"reasoning___a": "why"}, {"a": 1, "reasoning___a": "why", "source___a": [1]},
             {"name": "alpha", "qty": 3, "ok": True}, {"name": "Alpha!", "qty": 3.0, "ok": 1}, {"name": "beta", "qty": 30, "ok": False},
             {"a": "a" * 60}, {"a": "b" * 60}, {"a": [1]}, {"a": {"b": 1}}, {"a": "", "b": 0}, [], [1, 2], ["a"], [{"a": 1}]]
    for _ in range(60):
        d = {rng.choice(["a", "b", "c", "name", "qty", "reasoning___x", "source___y"]): rng.choice(pool[:60]) for _ in range(rng.randrange(0, 5))}
        pool.append(d)
    return pool


def edge_pairs():
    """Pairs on the boundaries the pass models: isclose at 1 % and one ulp past, big ints, 50 / 51 raw characters, 64 / 65
    normalised characters, empty normalised forms, falsy values, dict keys."""
    cases = []
    for base in (1.0, 100.0, 3.7, -2.5, 1e10, 7e-300):
        edge = base + abs(base) * 0.01
        cases += [(base, edge), (base, math.nextafter(edge, math.inf)), (base, math.nextafter(edge, -math.inf))]
        edge = base - abs(base) * 0.01
        cases += [(base, edge), (base, math.nextafter(edge, math.inf)), (base, math.nextafter(edge, -math.inf))]
    cases += [(100, 101), (100, 102), (100, 101.0), (100, 101.00000000001), (True, 1), (True, 1.0), (False, 0), (True, False),
              (10 ** 20, 10 ** 20), (10 ** 20, 10 ** 20 + 1), (10 ** 30, 10 ** 31), (-(10 ** 25), -(10 ** 25)), (2 ** 63, 2 ** 63 - 1),
              (0, 0.0), (0, ""), (0.0, False), ("", None), (None, {}), ({}, []), (None, []), (0, None), (None, None), (1, None),
              ("a" * 50, "b" * 50), ("a" * 51, "b" * 50), ("a" * 51, "b" * 51), ("a" * 51, "a" * 51),
              ("x" * 64, "y" * 70), ("x" * 65, "y" * 70), ("x" * 64 + "!", "x" * 64), ("!!!", "?"), ("!!!", "abc"), ("", "abc"),
              ("Hello, World", "hello world"), ("abc", 1), ("abc", {"a": 1}), ({"a": 1}, 1),
              ({"a": 1, "b": "x"}, {"c": 2, "d": "y"}), ({"a": 1, "b": "x"}, {"b": "x", "c": 2}), ({"a": 1, "reasoning___a": "z"}, {"a": 1}),
              ({"reasoning___a": "z"}, {}), ({"source___b": [1]}, {"source___b": 2}), ({"a": [1]}, {"a": [1]}), ({"a": {"b": 1}}, {"a": 1}),
              ({"a": "a" * 60}, {"a": "b" * 60}), ({"a": None}, {"b": None}), ({"a": 1.0}, {"a": True}), ([1], [1]), ([], [])]
    return cases


NODE_SIZES = (2, 3, 31, 32, 33, 63, 64, 65, 200, 511, 512)


def node_sets(rng):
    """List nodes for the batched pass (kc_debug_alignsim_nodes), shuffled: every size of NODE_SIZES (one lane's pair, a warp's
    pairs exactly, one more, several rows per step, the 512 limit), thousands of small nodes so that every warp of the grid takes
    several, and the edge pairs as nodes of two.  Returns (pool of distinct elements, [pool indices of each node's elements])."""
    pool = element_pool(rng)
    for a, b in edge_pairs():
        pool += [a, b]
    texts, uniq = set(), []
    for e in pool:  # one pool entry per JSON text
        t = json.dumps(e)
        if t not in texts:
            texts.add(t)
            uniq.append(e)
    index = {json.dumps(e): i for i, e in enumerate(uniq)}
    counts = {2: 2500, 3: 2500, 31: 1000, 32: 1000, 33: 1000, 63: 100, 64: 100, 65: 100, 200: 10, 511: 3, 512: 3}
    nodes = [[rng.randrange(len(uniq)) for _ in range(T)] for T in NODE_SIZES for _ in range(counts[T])]
    nodes += [[index[json.dumps(a)], index[json.dumps(b)]] for a, b in edge_pairs()]
    rng.shuffle(nodes)
    return uniq, nodes


def run_nodes(pool, nodes, lanes=1, device=-1):
    """kc_debug_alignsim_nodes over `nodes` (pool indices) -> (pairs decided, every node's matrix back to back, float64)."""
    import ctypes

    import numpy as np
    from k_llms_b200 import _native as K
    enc = [json.dumps(e).encode() for e in pool]
    flat = [enc[i] for nd in nodes for i in nd]
    texts = (ctypes.c_char_p * len(flat))(*flat)
    lens = np.array([len(nd) for nd in nodes], dtype=np.int32)
    # a NaN payload the pass never writes: a cell the host phase skips keeps it
    out = np.full(int((lens.astype(np.int64) ** 2).sum()), 0x7FF4DEAD0000BEEF, dtype=np.uint64).view(np.float64)
    rc = K.load().kc_debug_alignsim_nodes(ctypes.cast(texts, ctypes.c_void_p), lens.ctypes.data, len(nodes), lanes, device, out.ctypes.data)
    if rc < 0:
        K.check(rc)
    return rc, out


def expected_matrices(pool, nodes):
    """What the pass must write for `nodes`: generic_similarity (kc_debug_similarity_json) where it models the pair, NaN
    elsewhere and on the diagonal, every node's matrix back to back; and the number of modelled pairs a < b."""
    import ctypes

    import numpy as np
    from k_llms_b200 import _native as K
    from tests.test_alignsim_host_logic import models
    lib = K.load()
    enc = [json.dumps(e).encode() for e in pool]
    S = np.full((len(pool), len(pool)), np.nan)
    v = ctypes.c_double()
    for i in range(len(pool)):
        for j in range(len(pool)):
            if models(pool[i], pool[j]):
                assert lib.kc_debug_similarity_json(enc[i], enc[j], ctypes.byref(v)) == 0
                S[i, j] = v.value
    parts, modelled = [], 0
    for nd in nodes:
        idx = np.asarray(nd)
        E = S[np.ix_(idx, idx)]
        np.fill_diagonal(E, np.nan)
        parts.append(E.reshape(-1))
        modelled += int(np.count_nonzero(~np.isnan(E[np.triu_indices(len(nd), 1)])))
    return np.concatenate(parts), modelled


def assert_matrices(got, exp):
    """NaN exactly where exp has NaN, the same bits everywhere else."""
    import numpy as np
    nan = np.isnan(exp)
    bad = np.nonzero((np.isnan(got) != nan) | (~nan & (got.view(np.uint64) != exp.view(np.uint64))))[0]
    assert len(bad) == 0, (len(bad), bad[:10], got[bad[:10]], exp[bad[:10]])


def _perturb(rng, v):
    if isinstance(v, dict):
        return {k: _perturb(rng, x) for k, x in v.items() if rng.random() > 0.05}
    if isinstance(v, list):
        lst = [_perturb(rng, x) for x in v]
        r = rng.random()
        if r < 0.25:
            rng.shuffle(lst)
        elif r < 0.4 and lst:
            lst.pop(rng.randrange(len(lst)))
        return lst
    return v


def random_records(rng, count):
    """`count` records (lists of candidate values, freshly parsed) mixing: shuffled / truncated copies of one truth list,
    nested schemas with list fields (oracle.gen_golden), scalar and dict lists with duplicates, lists inside list elements,
    nodes of more than 512 elements, and lists holding two long strings (those records need the Python pre-pass)."""
    out = [c for c in random_list_records(rng.randrange(1 << 30), count // 5)]
    elems = element_pool(rng)
    small = [e for e in elems if not (isinstance(e, str) and len(e) > 50)]
    while len(out) < count:
        r = rng.random()
        if r < 0.3:
            cands = _record_candidates(rng, rng.choice([2, 3, 5, 8]), depth=3)
            out.append([_perturb(rng, c) if rng.random() < 0.85 else None for c in cands])
            continue
        n = rng.choice([2, 3, 4, 5, 8])
        if r < 0.75:
            base = [rng.choice(small) for _ in range(rng.randrange(0, 7))]
        elif r < 0.85:  # lists inside list elements
            base = [{"tags": [rng.choice(small) for _ in range(rng.randrange(0, 4))], "id": rng.randrange(5)} for _ in range(rng.randrange(1, 4))]
            if rng.random() < 0.5:
                base = [[rng.choice(small) for _ in range(rng.randrange(0, 3))] for _ in range(rng.randrange(1, 4))]
        elif r < 0.97:  # two long strings in one node
            base = [rng.choice(small) for _ in range(rng.randrange(0, 3))] + ["a" * 60 + str(rng.randrange(9)), "b" * 55]
        else:  # more than 512 elements in one node
            n = 3
            base = [rng.randrange(1000) for _ in range(rng.randrange(172, 200))]
        vals = []
        for _c in range(n):
            lst = json.loads(json.dumps(base))
            q = rng.random()
            if q < 0.3:
                rng.shuffle(lst)
            elif q < 0.5 and lst:
                lst.pop(rng.randrange(len(lst)))
            elif q < 0.6:
                lst.append(rng.choice(small))
            elif q < 0.63:
                lst = rng.choice([None, "not a list", 3])
            vals.append({"f": {"items": lst}, "k": rng.randrange(3)} if rng.random() < 0.6 else lst)
        out.append(vals)
    return [json.loads(json.dumps(v)) for v in out[:count]]
