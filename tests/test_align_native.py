"""H2 (kc_align_json: the alignment pre-pass in native host code) against the reference's own outputs
(tests/golden/alignment.json) and against the Python port of the pre-pass on random structures.  CPU only."""
import json
import logging
import random

import numpy as np
import pytest

from tests.helpers import load_golden, raising_embeddings


def _python_align(values):
    from k_llms_b200.utils.consensus_utils import recursive_list_alignments
    logging.disable(logging.CRITICAL)
    try:
        return recursive_list_alignments(json.loads(json.dumps(values)), "embeddings", raising_embeddings, None, 0.51)[0]
    finally:
        logging.disable(logging.NOTSET)


def test_alignment_goldens_reference_outputs():
    from k_llms_b200 import _native as K
    cases = load_golden("alignment")
    assert len(cases) > 100
    for case in cases:
        got = K.align_json(case["values"], 0.51)
        assert got is not None and json.dumps(got) == json.dumps(case["aligned"]), case["values"]


def test_alignment_matches_python_port_on_random_structures():
    from k_llms_b200 import _native as K
    from oracle.gen_golden import _record_candidates, random_list_records
    rng = random.Random(2026)
    cases = list(random_list_records(321, 250))

    def perturb(v):
        if isinstance(v, dict):
            return {k: perturb(x) for k, x in v.items() if rng.random() > 0.05}
        if isinstance(v, list):
            lst = [perturb(x) for x in v]
            r = rng.random()
            if r < 0.25:
                rng.shuffle(lst)
            elif r < 0.4 and lst:
                lst.pop(rng.randrange(len(lst)))
            return lst
        return v

    for _ in range(150):
        cands = _record_candidates(rng, rng.choice([2, 3, 5, 8]), depth=3)
        cases.append([perturb(c) if rng.random() < 0.85 else None for c in cands])
    # scalar lists: duplicates, None elements, values CPython shares between positions (identity quirk of majority_sorting.py)
    pool = [1, 2, 3, 5, 300, 300, 1000, "a", "b", "ab", "ab", "", True, False, None, 2.5, 2.5, "alpha", "alpha beta", [1, 2], [2, 1], {"k": [1]}]
    for _ in range(600):
        base = [rng.choice(pool) for _ in range(rng.randrange(0, 6))]
        vals = []
        for _c in range(rng.choice([2, 3, 4, 5, 8])):
            lst = json.loads(json.dumps(base))
            r = rng.random()
            if r < 0.3:
                rng.shuffle(lst)
            elif r < 0.5 and lst:
                lst.pop(rng.randrange(len(lst)))
            elif r < 0.6:
                lst.append(rng.choice(pool))
            elif r < 0.65:
                lst = rng.choice([None, "not a list", 3])
            vals.append({"tags": lst} if rng.random() < 0.6 else lst)
        cases.append(vals)
    for values in cases:
        values = json.loads(json.dumps(values))  # what consolidation.py passes: freshly parsed values (align_json declines lists
        got = K.align_json(values, 0.51)         # that hold one longer string / float object twice: object identity matters upstream)
        assert got is not None
        assert json.dumps(got) == json.dumps(_python_align(values)), values


def test_alignment_declines_what_needs_embeddings_or_unicode():
    from k_llms_b200 import _native as K
    assert K.align_json([["a" * 60, "x"], ["b" * 60, "x"]], 0.51) is None       # cu:813: both strings > 50 characters
    assert K.align_json([["café"], ["cafe"]], 0.51) is None
    assert K.align_json([["a" * 60, "x"], ["short", "x"]], 0.51) is not None


def test_assignment_solver_is_scipys():
    from scipy.optimize import linear_sum_assignment
    from k_llms_b200 import _native as K
    lib = K.load()
    rng = np.random.default_rng(0)
    for it in range(3000):
        nr, nc = int(rng.integers(1, 9)), int(rng.integers(1, 9))
        cost = [rng.random((nr, nc)), rng.integers(0, 3, (nr, nc)).astype(float), np.full((nr, nc), 0.5),
                1.0 - rng.choice([1e-8, 1.0, 0.5, 0.75], (nr, nc)), np.round(rng.random((nr, nc)), 1)][it % 5]
        cost = np.ascontiguousarray(cost, dtype=np.float64)
        er, ec = linear_sum_assignment(cost)
        a, b = np.zeros(8, np.int32), np.zeros(8, np.int32)
        k = lib.kc_debug_lsap(nr, nc, cost.ctypes.data, a.ctypes.data, b.ctypes.data)
        assert k == len(er) and np.array_equal(a[:k], er) and np.array_equal(b[:k], ec), cost


def test_native_similarity_matches_python():
    import ctypes
    from k_llms_b200 import _native as K
    from k_llms_b200.utils import similarity as S
    lib = K.load()
    rng = random.Random(3)
    words = ["alpha", "Bravo", "charlie delta", "x", "", "The Quick brown fox", "the quick brown fax", "12 apples", "N/A"]

    def rand_val(d=0):
        r = rng.random()
        if r < 0.1:
            return None
        if r < 0.2:
            return rng.random() < 0.5
        if r < 0.35:
            return rng.choice([0, 1, 2, 100, 101, -5, 10 ** 20, 99, 1000])
        if r < 0.5:
            return rng.choice([0.0, 1.0, 1.005, 2.5, 100.9, -0.0, 1e-9, 3.14159])
        if r < 0.7:
            return rng.choice(words)
        if d < 3 and r < 0.85:
            return [rand_val(d + 1) for _ in range(rng.randrange(0, 4))]
        if d < 3:
            return {rng.choice(["a", "b", "c", "reasoning___x", "source___y", "name"]): rand_val(d + 1) for _ in range(rng.randrange(0, 4))}
        return 1

    pairs = []
    for _ in range(4000):
        a, b = rand_val(), rand_val()
        if rng.random() < 0.3:
            b = json.loads(json.dumps(a))
        pairs.append((a, b))
    # a decoded string's backslash before a letter is a character, not an escape: "x\\ty" normalises to "xty"
    pairs += [("x\\ty", "xty"), ("x\\ty", "x\ty"), (["a\\b c"], ["ab c"]), ({"name": "n\\nb"}, {"name": "nnb"})]
    for a, b in pairs:
        S._cache.clear()
        exp = float(S.generic_similarity(a, b, "embeddings", raising_embeddings))
        out = ctypes.c_double()
        rc = lib.kc_debug_similarity_json(json.dumps(a).encode(), json.dumps(b).encode(), ctypes.byref(out))
        assert rc == 0 and abs(out.value - exp) <= 1e-12, (a, b, exp, out.value)


def test_consolidation_uses_the_native_prepass_with_identical_results():
    """The hook consolidation.py calls before the vote: same aligned contents as the Python pre-pass on every client-order
    golden input, and None (Python fallback) for the non-default similarity methods."""
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from k_llms_b200.utils.consolidation import _native_alignment
    used = 0
    for case in load_golden("client_order"):
        contents = json.loads(json.dumps(case["values"]))
        native = _native_alignment(contents, ConsensusSettings())
        assert native is not None
        used += 1
        assert json.dumps(native) == json.dumps(_python_align(contents))
    assert used > 100
    assert _native_alignment([{"a": [1]}, {"a": [1]}], ConsensusSettings(string_similarity_method="jaccard")) is None


def test_align_json_declines_values_with_shared_object_identity():
    """ADVICE r1: the native alignment assumes json.loads-like object identity; a list holding the same string object twice
    (built in Python) goes to the Python pre-pass instead of being aligned on that assumption."""
    import json
    from k_llms_b200 import _native as K
    w = "gadget"
    shared = [{"items": [w, "widget", w]}, {"items": ["widget", w]}]  # the SAME str object twice in one list
    assert K.align_json(shared, 0.51) is None
    fresh = [json.loads(json.dumps(v)) for v in shared]                # what consolidation.py passes: freshly parsed
    assert K.align_json(fresh, 0.51) is not None
