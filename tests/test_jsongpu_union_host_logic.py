"""The device JSON path's key-union round (U1-U3, k_llms_b200/csrc/kc_jsongpu.cuh) on a machine without a GPU: records whose
candidates order their keys differently, lack keys, hold extra ones or hold None (or nothing) where others hold a sub-object.
The host instantiation of the phases (kc_debug_jsongpu_plan_flags with KC_JSON_KEY_UNION) runs the union round lane by lane with
the oracle in the kernels' place; every such record must come out on the device path, byte-identical to the reference's client
order, and every record the round cannot model exactly must be declined with the same reason the rest of the device path gives.
Without the flag the phases decline these records exactly as before."""
import json
import random

import numpy as np
import pytest

from k_llms_b200._native import JSON_KEY_UNION, JSON_NUMERIC_MEDOID
from oracle import consensus_py as O
from tests import weighted_oracle as W
from tests.helpers import jsongpu_with_oracle
from tests.test_async_native_host_logic import oracle_kernels, python_async  # noqa: F401  (a fixture)
from tests.test_gpu_json import _expected
from tests.test_weighted_host_logic import EMBED

KEYS = ["zeta", "Alpha", "b", "a", "aa", "k1", "k10", "k2", "Z", "id", "name", "addr"]
# short phrases only: two strings over 50 characters are the embeddings service's, which every path declines
UPHRASES = ["the quick brown fox", "The Quick Brown Fox!", "the quick brown fax", "a quick brown fox jumps", "net 30 days",
            "Net 30 Days.", "payment due on receipt", "- - -", "x y z"]
EXTRA = {"x_int": lambda rng: rng.randrange(0, 50), "x_enum": lambda rng: rng.choice(["alpha", "Bravo", "ALPHA!"]),
         "x_bool": lambda rng: rng.random() < 0.5, "x_float": lambda rng: rng.choice([1.5, 2.25, 1.5000001])}


def union_record(rng, n, p_shuffle=0.5, p_drop=0.15, p_extra=0.15, p_null=0.15):
    """n candidates of one schema (objects up to depth 4, like _shaped_record) that each reorder their members at every
    level, drop keys, add extra keys and set sub-objects to None or drop them, independently.  Now and then candidate 0 keeps
    only one top-level key, a key is in every candidate but candidate 0, or a phrase is in one candidate only."""
    def shape(depth):
        out = []
        for k in rng.sample(KEYS, rng.randrange(1, 6)):
            if depth < 4 and rng.random() < 0.35:
                out.append((k, shape(depth + 1)))
            else:
                out.append((k, rng.choice(["enum", "bool", "int", "float", "phrase", "allnull", "one"])))
        return out

    def truth_of(sh):
        return [(k, truth_of(v) if isinstance(v, list) else
                 {"enum": lambda: rng.choice(["alpha", "Bravo", "two words", ""]), "bool": lambda: rng.random() < 0.5,
                  "int": lambda: rng.randrange(-5, 10 ** rng.randrange(1, 7)), "float": lambda: round(rng.uniform(-10, 1e4), 6),
                  "phrase": lambda: rng.choice(UPHRASES), "allnull": lambda: None, "one": lambda: rng.choice([7, "solo", 2.5])}[v]())
                for k, v in sh]

    def leaf(kind, tv, c):
        v, r = tv, rng.random()
        if kind == "one":
            return v if c == 0 else None
        if r < 0.3:
            return {"enum": lambda: rng.choice(["ALPHA", "bravo!", "x"]), "bool": lambda: rng.random() < 0.5,
                    "int": lambda: rng.randrange(0, 100), "float": lambda: round(rng.uniform(0, 10), 6), "phrase": lambda: rng.choice(UPHRASES),
                    "allnull": lambda: None}[kind]()
        return None if r > 0.92 else v

    def candidate(sh, tr, c, depth, lone):
        items = []
        for (k, kind), (_k, tv) in zip(sh, tr):
            if rng.random() < p_drop:
                continue
            if isinstance(kind, list):
                items.append((k, None if rng.random() < p_null else candidate(kind, tv, c, depth + 1, lone)))
            else:
                items.append((k, leaf(kind, tv, c)))
        for name, draw in EXTRA.items():
            if rng.random() < p_extra / len(EXTRA):
                items.append((name, draw(rng)))
        if depth == 1 and lone and c == lone[0]:
            items.append(("x_phrase", rng.choice(UPHRASES)))
        if not items:  # empty objects are declined everywhere: keep one member
            (k, kind), (_k, tv) = sh[0], tr[0]
            items.append((k, None if isinstance(kind, list) else leaf(kind, tv, c)))
        if rng.random() < p_shuffle:
            rng.shuffle(items)
        return dict(items)

    sh = shape(1)
    tr = truth_of(sh)
    lone = [rng.randrange(n)] if rng.random() < 0.15 else None
    cands = [candidate(sh, tr, c, 1, lone) for c in range(n)]
    r = rng.random()
    if r < 0.1:                     # every key of candidate 0 but one
        k = rng.choice(list(cands[0]))
        cands[0] = {k: cands[0][k]}
    elif r < 0.2:                   # a key only candidate 0 lacks
        for c in range(1, n):
            cands[c]["x_others"] = rng.randrange(0, 3)
    return [json.dumps(d) for d in cands]


def union_records(seed, count, ns=(2, 3, 5, 8, 16, 33, 64)):
    rng = random.Random(seed)
    by_n = {}
    for _ in range(count):
        n = rng.choice(ns)
        by_n.setdefault(n, []).append(union_record(rng, n))
    return by_n


def _differ_in_shape(texts):
    """Whether the candidates' key sequences differ (so the record needs the union round)."""
    def keys(v):
        return [(k, keys(x) if isinstance(x, dict) else None) for k, x in v.items()]
    return len({json.dumps(keys(json.loads(t))) for t in texts}) > 1


def test_union_records_on_the_device_path():
    on_union = 0
    for _n, recs in union_records(101, 1400).items():
        pairs, status = jsongpu_with_oracle(recs, flags=JSON_KEY_UNION)
        for texts, got, st in zip(recs, pairs, status):
            assert st == 0, (texts, st)
            on_union += _differ_in_shape(texts)
            assert got == _expected(texts), texts
    assert on_union > 1000, on_union


def test_union_records_under_the_async_medoid(oracle_kernels):  # noqa: F811
    for _n, recs in union_records(202, 500, ns=(2, 3, 5, 8, 16)).items():
        pairs, status = jsongpu_with_oracle(recs, flags=JSON_KEY_UNION | JSON_NUMERIC_MEDOID)
        for texts, got, st in zip(recs, pairs, status):
            assert st == 0, (texts, st)
            assert got == python_async(texts), texts


def test_union_records_weighted():
    rng = np.random.default_rng(7)
    for _n, recs in union_records(303, 500, ns=(2, 3, 5, 8, 16, 33)).items():
        n = len(recs[0])
        seq = (-rng.exponential(4.0, len(recs) * n)).astype(np.float32)
        seq[:n] = -1.5  # equal sums: the count winner
        pairs, status = jsongpu_with_oracle(recs, seq, flags=JSON_KEY_UNION)
        for r, (texts, got, st) in enumerate(zip(recs, pairs, status)):
            assert st == 0, (texts, st)
            contents = [json.loads(t) for t in texts]
            value, conf = W.client_order(contents, seq[r * n:(r + 1) * n], O.DEFAULTS, EMBED)
            assert got == (json.dumps(value), json.dumps(conf)), (texts, got, value, conf)


def test_same_shape_records_are_untouched_and_mixed_batches_agree():
    """One batch of union records interleaved with same-shape records gives each record what it gives alone."""
    from tests.test_jsongpu_host_logic import _shaped_record
    rng = random.Random(9)
    recs = []
    for i in range(300):
        recs.append(_shaped_record(rng, 5) if i % 3 else union_record(rng, 5))
    pairs, status = jsongpu_with_oracle(recs, flags=JSON_KEY_UNION)
    for texts, got, st in zip(recs, pairs, status):
        alone, st1 = jsongpu_with_oracle([texts], flags=JSON_KEY_UNION)
        assert (got, st) == (alone[0], st1[0]), texts
        if got is not None:
            assert got == _expected(texts)


WIDE = json.dumps({f"k{i:03d}": i for i in range(600)}), json.dumps({f"j{i:03d}": i for i in range(600)})

ACCEPTED = {
    "key order differs": ['{"a": 1, "b": 2}', '{"b": 2, "a": 1}'],
    "keys differ": ['{"a": 1, "b": 2}', '{"a": 1}'],
    "nested here, None there": ['{"a": {"b": 1}}', '{"a": null}'],
    "nested here, missing there": ['{"a": {"b": {"c": true}}, "d": 1}', '{"d": 2}', '{"d": 1, "a": null}'],
    "nested keys differ": ['{"a": {"b": 1}}', '{"a": {"c": 1}}'],
    "nested shapes differ": ['{"a": {"b": 1}, "c": 2}', '{"a": {"b": 1, "c": 2}}'],
    "candidate 0 lacks the key": ['{"a": 1}', '{"a": 1, "zz": "x"}', '{"zz": "y", "a": 2}'],
    "text is not the whole union": ['{"text": "x"}', '{"text": "y", "extra": null}'],
    "a phrase in one candidate": ['{"a": 1}', '{"a": 1, "p": "the quick brown fox"}', '{"a": 2}'],
    "all-null leaf from the union": ['{"a": 1, "n": null}', '{"a": 1}'],
}

DECLINED = {  # name: (texts, D_* code)
    "object against 0": (['{"a": {"b": 1}, "c": 1}', '{"c": 1, "a": 0}'], 4),
    "object against a string, reordered": (['{"c": 1, "a": "x"}', '{"a": {"b": 1}, "c": 1}'], 4),
    "object against a list": (['{"a": {"b": 1}}', '{"a": [1]}'], 4),
    "empty object in one candidate": (['{"a": 1}', '{}'], 13),
    "empty nested object in one candidate": (['{"a": {"b": 1}, "c": 1}', '{"c": 1, "a": {}}'], 4),
    "duplicate key in one candidate, absent in the other": (['{"a": 1, "b": 2, "b": 3}', '{"a": 1}'], 8),
    "nested duplicate key, reordered": (['{"x": {"b": 1, "b": 2}, "a": 1}', '{"a": 1}'], 8),
    "reasoning key in one candidate only": (['{"a": 1, "reasoning___x": "y"}', '{"a": 2}'], 9),
    "text is the whole record": (['{"text": "x"}', '{"text": "y"}'], 9),
    "union above 1024 tokens": (list(WIDE), 7),
    "nine levels in one candidate": (['{"b": 1}', '{"b": 1, "a": ' + '{"a": ' * 9 + '1' + '}' * 10], 4),
    "mixed types across the union": (['{"a": "x", "b": 1}', '{"b": 1}', '{"a": 3}'], 11),
    "unicode escape in a reordered candidate": (['{"a": "x", "b": 1}', '{"b": 1, "a": "\\u0041"}'], 3),
    "broken text next to a reordered one": (['{"a": 1, "b": 2}', '{"b": 2, "a": 1}', '{"a": 1, "b": 2'], 2),
    "number out of range, reordered": (['{"a": 1, "b": 2}', '{"b": 1e999, "a": 1}'], 12),
}


@pytest.mark.parametrize("name", list(ACCEPTED))
def test_union_edge_accepted(name):
    texts = ACCEPTED[name]
    (got,), (st,) = jsongpu_with_oracle([texts], flags=JSON_KEY_UNION)
    assert st == 0 and got == _expected(texts), (name, st, got)


@pytest.mark.parametrize("name", list(DECLINED))
def test_union_edge_declined(name):
    texts, why = DECLINED[name]
    (got,), (st,) = jsongpu_with_oracle([texts], flags=JSON_KEY_UNION)
    assert got is None and st == why, (name, st)


def test_declines_what_it_does_not_model_after_the_union():
    """The cases the device path still declines, one batch: none of them may come back with an internal status."""
    cases = {
        "unicode escape": ['{"a": "x\\u0041y"}', '{"a": "x"}'],
        "escape in a key": ['{"a\\n": "x"}', '{"a\\n": "x"}'],
        "bad escape": ['{"a": "x\\qy"}', '{"a": "x"}'],
        "non-ascii": ['{"a": "café"}', '{"a": "cafe"}'],
        "nested here, scalar there": ['{"a": {"b": 1}}', '{"a": 3}'],
        "empty nested object": ['{"a": {}}', '{"a": {}}'],
        "nested duplicate key": ['{"a": {"b": 1, "b": 2}}', '{"a": {"b": 1, "b": 2}}'],
        "nested special key": ['{"a": {"reasoning___b": "x", "c": 1}}', '{"a": {"reasoning___b": "y", "c": 1}}'],
        "list in a nested object": ['{"a": {"b": [1]}}', '{"a": {"b": [1]}}'],
        "nine levels": ['{"a": ' * 10 + '1' + '}' * 10] * 2,
        "list": ['{"a": [1, 2]}', '{"a": [1, 2]}'],
        "duplicate key": ['{"a": 1, "a": 2}', '{"a": 1, "a": 2}'],
        "free text": ["hello there", "hello there"],
        "top-level list": ["[1, 2]", "[1, 2]"],
        "nan": ['{"a": NaN}', '{"a": 1}'],
        "two long phrases": ['{"a": "%s"}' % ("the big cat " * 5), '{"a": "%s"}' % ("the big dog " * 5)],
        "phrase and number": ['{"a": "the big cat"}', '{"a": 3}'],
        "mixed str": ['{"a": "x"}', '{"a": 3}'],
        "text wrapper": ['{"text": "x"}', '{"text": "x"}'],
        "reasoning key": ['{"reasoning___a": "x", "b": 1}', '{"reasoning___a": "y", "b": 1}'],
        "empty object": ["{}", "{}"],
        "20 digits": ['{"a": 123456789012345678901}', '{"a": 1}'],
        "trailing junk": ['{"a": 1} x', '{"a": 1}'],
        "empty content": ['{"a": 1}', ''],
    }
    pairs, status = jsongpu_with_oracle(list(cases.values()), flags=JSON_KEY_UNION)
    for (name, _), got, st in zip(cases.items(), pairs, status):
        assert got is None and 0 < st < 0xFF, (name, st)


def test_without_the_flag_nothing_changes():
    """The same records without KC_JSON_KEY_UNION: the records whose candidates differ in shape are declined with the reasons A1
    gave before the union round existed, and every other record comes out as it does with the flag."""
    recs = [t for _n, group in union_records(404, 300, ns=(3,)).items() for t in group]
    with_flag, st_flag = jsongpu_with_oracle(recs, flags=JSON_KEY_UNION)
    without, st = jsongpu_with_oracle(recs)
    declined = 0
    for texts, a, b, s_flag, s in zip(recs, with_flag, without, st_flag, st):
        if _differ_in_shape(texts):
            declined += 1
            assert b is None and s in (4, 7), (texts, s)   # D_NESTED, D_KEYS_DIFFER
        else:
            assert (a, s_flag) == (b, s), texts
    assert declined > 200, declined
    for name, texts in ACCEPTED.items():
        (got,), (s,) = jsongpu_with_oracle([texts])
        assert got is None and s in (4, 7), (name, s)
