"""GPU parity for H1 (native JSON in -> consensus JSON out): byte-identical to the reference's client order
(align + consensus + json.dumps), which the object-level oracle restates (oracle/consensus_py.client_order)."""
import json
import random

import pytest

from oracle import consensus_py as O
from tests.helpers import raising_embeddings

pytestmark = pytest.mark.gpu

PHRASE_WORDS = "invoice total due amount net gross payment bank transfer within thirty days from receipt of goods acme corp ltd".split()


def _phrase(rng, lo=3, hi=8):
    return " ".join(rng.choice(PHRASE_WORDS) for _ in range(rng.randrange(lo, hi + 1)))


def _phrase_variant(rng, base):
    words = base.split()
    r = rng.random()
    if r < 0.3:
        words[rng.randrange(len(words))] = rng.choice(PHRASE_WORDS)
    elif r < 0.5:
        words = words[:-1] if len(words) > 1 else words     # may leave fewer than three words
    elif r < 0.7:
        words = [w.upper() if rng.random() < 0.5 else w + "," for w in words]
    elif r < 0.8:
        return _phrase(rng, 12, 16)                         # one long candidate (> 50 characters) stays inside K4's contract
    return " ".join(words)


WORDS = ["alpha", "Bravo", "charlie", "DELTA", "echo", "fox-trot", "golf", "Hotel", "", "a b", "x\ty", 'q"uote', "back\\slash", "nl\n"]

# Records at n = 3 on the edges of the text rules: DEL (json.dumps prints it as \u007f) in a vote string, a medoid string, a key
# and free text inside the {"text": ...} wrapper; a literal backslash before a letter in free text and in a list record's string
# (decoded values: the backslash is a character, "x\\ty" sanitises to "xty")
TEXT_EDGES = [
    ['{"s": "x\x7fy"}', '{"s": "x\x7fy"}', '{"s": "xy"}'],
    ['{"p": "one two\x7f three"}', '{"p": "one two\x7f three"}', '{"p": "one two four"}'],
    ['{"k\x7f": "x", "b": 1}', '{"k\x7f": "x", "b": 2}', '{"k\x7f": "y"}'],
    ['x\x7fy "q" \\', '{"text": "x\x7fy \\"q\\" \\\\", "b": 1}', 'x\x7fy "q" \\'],
    ['x\\ty', 'x\\ty', '{"text": "xty"}'],
    ['{"s": "x\\\\ty", "l": [1]}', '{"s": "x\\\\ty", "l": [1]}', '{"s": "xty", "l": [1]}'],
]


def _expected(texts):
    from k_llms_b200.utils.consolidation import _format_consensus_content, _safe_parse_content
    contents = [_safe_parse_content(t) for t in texts if t]
    value, conf = O.client_order(contents, embed=raising_embeddings)
    return _format_consensus_content(value), json.dumps(conf)


def _random_record(rng, n):
    n_fields = rng.randrange(1, 7)
    kinds = [rng.choice(["str", "bool", "int", "float", "near", "big", "mixnum", "phrase", "phrase"]) for _ in range(n_fields)]
    truth = {}
    for f, k in enumerate(kinds):
        truth[f] = {"str": lambda: rng.choice(WORDS), "bool": lambda: rng.random() < 0.5,
                    "int": lambda: rng.randrange(-50, 10 ** rng.randrange(1, 8)), "float": lambda: rng.uniform(-1e3, 1e5),
                    "near": lambda: rng.choice([1.0, 100.0, 1e-5, 1e16, 123456789.125, 0.0, -0.0]),
                    "big": lambda: rng.choice([10 ** 30, 2 ** 63, -(10 ** 25), 10 ** 400]),
                    "mixnum": lambda: rng.choice([1, 1.0, 2, 2.5]), "phrase": lambda: _phrase(rng)}[k]()
    texts = []
    for _ in range(n):
        d = {}
        for f, k in enumerate(kinds):
            r = rng.random()
            if r < 0.08:
                continue  # key missing
            v = truth[f]
            if r < 0.3:
                v = {"str": lambda: rng.choice(WORDS).upper(), "bool": lambda: rng.random() < 0.5,
                     "int": lambda: rng.randrange(0, 1000), "float": lambda: rng.uniform(0, 10),
                     "near": lambda: truth[f] * rng.choice([1.02, 0.97, 1.05, 10.0]) if isinstance(truth[f], float) else 3.0,
                     "big": lambda: rng.choice([10 ** 30 + 1, 7]), "mixnum": lambda: rng.choice([True, "1", None, 3]),
                     "phrase": lambda: _phrase_variant(rng, truth[f])}[k]()
            if r > 0.93:
                v = None
            d[f"k{f}" if rng.random() > 0.02 else "reasoning___why"] = v
        t = json.dumps(d)
        if rng.random() < 0.03:
            t = t.replace(", ", " ,\n ")  # odd whitespace
        texts.append(t)
    return texts


def _random_nested_record(rng, n, depth=0):
    """Candidates sharing a schema of nested objects (no lists): missing / null sub-objects, empty objects, leaf fields of
    every kind, and now and then a candidate whose sub-object is a scalar or a list (the native path must decline those)."""
    def schema(d):
        out = {}
        for f in range(rng.randrange(1, 5)):
            r = rng.random()
            if d < 3 and r < 0.35:
                out[f"o{f}"] = schema(d + 1)
            else:
                out[f"k{f}"] = rng.choice(["str", "bool", "int", "float", "phrase"])
        return out

    def truth_of(sc):
        return {k: (truth_of(v) if isinstance(v, dict) else
                    {"str": lambda: rng.choice(WORDS), "bool": lambda: rng.random() < 0.5, "int": lambda: rng.randrange(0, 500),
                     "float": lambda: round(rng.uniform(0, 100), 2), "phrase": lambda: _phrase(rng)}[v]()) for k, v in sc.items()}

    def noisy(sc, tr):
        out = {}
        for k, v in sc.items():
            r = rng.random()
            if r < 0.07:
                continue
            if r < 0.12:
                out[k] = None
                continue
            if isinstance(v, dict):
                out[k] = {} if rng.random() < 0.05 else noisy(v, tr[k])
            elif rng.random() < 0.25:
                out[k] = {"str": lambda: rng.choice(WORDS).upper(), "bool": lambda: rng.random() < 0.5, "int": lambda: rng.randrange(0, 500),
                          "float": lambda: round(rng.uniform(0, 100), 2), "phrase": lambda: _phrase_variant(rng, tr[k])}[v]()
            else:
                out[k] = tr[k]
        return out

    sc = schema(0)
    tr = truth_of(sc)
    return [json.dumps(noisy(sc, tr)) for _ in range(n)]


def test_native_json_nested_objects():
    """Nested objects (no lists) stay on the native path: sorted keys and None fill at every level, nested output."""
    from k_llms_b200 import _native as K
    rng = random.Random(77)
    by_n = {}
    for _ in range(1500):
        n = rng.choice([2, 3, 5, 8])
        by_n.setdefault(n, []).append(_random_nested_record(rng, n))
    specials = [
        ['{"a": {"b": 1, "c": {"d": "x"}}}', '{"a": {"b": 1, "c": {"d": "X!"}}}', '{"a": null}'],
        ['{"a": {}}', '{"a": {}}'], ['{"a": {"b": {}}}', '{"a": {}}', '{}'],
        ['{"a": {"b": 1}, "a": {"b": 2}}', '{"a": {"b": 2}}'],                       # duplicate key: the last object wins
        ['{"a": {"reasoning___x": {"deep": [1, 2]}, "v": 3}}', '{"a": {"v": 3}}'],     # skipped key holding a list
        ['{"a": {"b": tru}}', '{"a": {"b": true}}', '{"a": {"b": true}}'],            # malformed inner value: whole text is free text
        ['{"text": {"text": "x"}}', '{"text": {"text": "x"}}'],
    ]
    for sp in specials:
        by_n.setdefault(len(sp), []).append(sp)
    native = nested_native = 0
    for n, recs in by_n.items():
        out = K.consolidate_json(recs)
        for texts, got in zip(recs, out):
            if got is None:
                continue
            native += 1
            nested_native += '": {' in got[0]
            exp = _expected(texts)
            assert got[0] == exp[0] and got[1] == exp[1], (texts, got, exp)
    assert native > 1200 and nested_native > 600
    declined = [['{"a": {"b": 1}}', '{"a": 5}'], ['{"a": {"b": 1}}', '{"a": [1]}']]  # a key mixing objects with other types
    assert K.consolidate_json(declined) == [None] * len(declined)


def _expected_with_lists(texts):
    """Client order incl. the list alignment: the Python pre-pass (pinned on the reference's alignment goldens) + the
    object-level oracle for the consensus."""
    import logging
    from k_llms_b200.utils.consensus_utils import recursive_list_alignments
    from k_llms_b200.utils.consolidation import _format_consensus_content, _safe_parse_content
    contents = [_safe_parse_content(t) for t in texts if t]
    logging.disable(logging.CRITICAL)
    try:
        aligned, _ = recursive_list_alignments(contents, "embeddings", raising_embeddings, None, 0.51)
    finally:
        logging.disable(logging.NOTSET)
    value, conf = O.consensus([(d if isinstance(d, dict) else {}) for d in aligned], embed=raising_embeddings)
    return _format_consensus_content(value), json.dumps(conf)


def test_native_json_list_fields():
    """Records with list fields stay native: the alignment pre-pass (H2) runs on the parsed tree, the merge is element-wise.
    Checked against the reference's own client-order outputs (goldens) and against the Python pre-pass + oracle."""
    from k_llms_b200 import _native as K
    from oracle.gen_golden import _record_candidates, random_list_records
    from tests.helpers import load_golden
    from k_llms_b200.utils.consolidation import _format_consensus_content
    by_n, native = {}, 0
    for case in load_golden("client_order"):
        if len(case["values"]) >= 2:
            by_n.setdefault(len(case["values"]), []).append(([json.dumps(v) for v in case["values"]], case))
    for n, items in by_n.items():
        for (texts, case), got in zip(items, K.consolidate_json([t for t, _ in items])):
            assert got is not None, texts
            native += 1
            assert got == (_format_consensus_content(case["value"]), json.dumps(case["conf"])), (texts, got)
    assert native > 100
    rng = random.Random(5)
    recs = [[json.dumps(v) for v in r] for r in random_list_records(77, 400)]
    for _ in range(200):
        recs.append([json.dumps(c) for c in _record_candidates(rng, rng.choice([2, 3, 5, 8]), depth=3)])
    by_n = {}
    for r in recs:
        by_n.setdefault(len(r), []).append(r)
    for n, rs in by_n.items():
        for texts, got in zip(rs, K.consolidate_json(rs)):
            assert got is not None and got == _expected_with_lists(texts), texts


def test_native_json_matches_reference_client_order():
    from k_llms_b200 import _native as K
    rng = random.Random(2024)
    records = []
    for _ in range(3000):
        n = rng.choice([2, 3, 5, 8, 16])
        records.append((n, _random_record(rng, n)))
    specials = [
        ['{"a": 1}', 'not json', '{"a": 1}'],                    # one candidate falls back to {"text": ...}
        ['Yes', 'yes', 'No'],                                    # free text: wrapper and unwrapping
        ['{"a": 1, "a": 2}', '{"a": 2}', '{"a": 1}'],            # duplicate keys: last one wins
        ['{}', '{}'], ['{"x": null}', '{"x": null}'],
        ['{"a": NaN, "b": Infinity}', '{"a": 1.5, "b": 2}', '{"a": 1.5, "b": 2}'],
        ['{"f": 1e400}', '{"f": 3}', '{"f": 3}'], ['{"f": 1E5}', '{"f": 100000.0}', '{"f": 1e+5}'],
        ['{"s": "a\\u0041b"}', '{"s": "aAb"}'], ['{"v": 0.1}', '{"v": 0.1}', '{"v": 0.30000000000000004}'],
        ['{"t": true, "u": "true"}', '{"t": null, "u": true}', '{"t": false, "u": "TRUE!"}'],
        ['{"p": "the big cat"}', '{"p": "the big cat"}', '{"p": "the big dog"}'],                  # medoid on K4
        ['{"p": "the big cat"}', '{"p": null}', '{}'],                                              # one non-None phrase
        ['{"p": "the big cat sat"}', '{"p": "a b"}', '{"p": ""}', '{"p": "THE BIG CAT SAT!"}'],     # short and empty members
        ['{"p": "one two three", "q": "x y z w"}', '{"p": "one two tree", "q": "x y z"}', '{"q": "x y z w"}'],
    ] + TEXT_EDGES
    for s in specials:
        records.append((len(s), s))
    by_n = {}
    for n, texts in records:
        by_n.setdefault(n, []).append(texts)
    native_count = 0
    for n, recs in by_n.items():
        out = K.consolidate_json(recs)
        assert len(out) == len(recs)
        for texts, got in zip(recs, out):
            if got is None:
                continue  # handed to the Python path by design (nested / multi-word / mixed bool groups ...)
            native_count += 1
            exp = _expected(texts)
            assert got[0] == exp[0], (texts, got, exp)
            assert got[1] == exp[1], (texts, got, exp)
    assert native_count > 2500


def test_native_json_declines_what_it_cannot_express():
    from k_llms_b200 import _native as K
    long1, long2 = " ".join(["payment"] * 9), " ".join(["transfer"] * 8)
    recs = [['{"a": [1, 2]}', '{"a": {"b": 1}}'], ['{"a": "one two three"}', '{"a": 7}'],
            [json.dumps({"a": long1}), json.dumps({"a": long2})],  # two strings > 50 chars: an embeddings pair
            ['{"a": "caf\\u00e9"}', '{"a": "cafe"}'], ['[1, 2]', '{"a": 1}'], ['', '{"a": 1}'], ['{"a": true}', '{"a": 1}']]
    assert K.consolidate_json(recs) == [None] * len(recs)
    ok = K.consolidate_json([['{"a": "x"}', '{"a": "X!"}']])
    assert ok == [('{"a": "x"}', '{"a": 1.0}')]


def test_batch_helper_mixes_native_and_python_paths():
    from k_llms_b200.utils.consolidation import consolidate_contents_batch
    records = [
        ['{"a": "x", "n": 5}', '{"a": "X!", "n": 5}', '{"a": "y", "n": 50}'],                 # native
        ['{"a": {"b": [1, 2]}}', '{"a": {"b": [1, 2]}}', '{"a": {"b": [2, 1]}}'],               # nested + list alignment: native (H2)
        ['{"a": {"b": 1}}', '{"a": 5}', '{"a": {"b": 1}}'],                                     # object vs scalar under one key: Python path
        ['{"t": "the big cat"}', '{"t": "the big cat"}', '{"t": "the big dog"}'],               # multi-word: medoid on the host
        ['Yes', 'yes', 'No'],
    ]
    out = consolidate_contents_batch(records)
    for texts, (content, lik) in zip(records, out):
        exp_content, exp_lik = _expected_full(texts)
        assert content == exp_content and lik == exp_lik, (texts, content, lik, exp_content, exp_lik)


def _expected_full(texts):
    """Expected output through the golden-pinned Python product path (align incl. lists + consensus)."""
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from k_llms_b200.utils.consolidation import _consensus_sync, _format_consensus_content, _safe_parse_content
    value, lik = _consensus_sync([_safe_parse_content(t) for t in texts], ConsensusSettings(), raising_embeddings, None)
    return _format_consensus_content(value), lik
