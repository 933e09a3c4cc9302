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
