"""The batched alignment pre-pass with its element similarities on the device (kc_align_json_batch, kc_alignsim.cuh): equal to
the per-record host alignment (kc_align_json), and the JSON consolidation entries that use it equal to the host logic
checked against the C oracle."""
import json
import random

import pytest

from tests.alignsim_cases import random_records
from tests.helpers import consolidate_json_with_oracle, load_golden

pytestmark = pytest.mark.gpu


def _check(records, min_support_ratio=0.51):
    from k_llms_b200 import _native as K
    counts = {}
    got = K.align_json_batch(records, min_support_ratio, device=0, counts=counts)
    assert len(got) == len(records)
    for values, g in zip(records, got):
        exp = K.align_json(values, min_support_ratio)
        assert (g is None) == (exp is None), values
        if exp is not None:
            assert json.dumps(g) == json.dumps(exp), values
    return got, counts


def _config3(rng, count, n=8):
    from oracle.gen_golden import _record_candidates
    return [json.loads(json.dumps(_record_candidates(rng, n, depth=3))) for _ in range(count)]


def _has_list(v):
    if isinstance(v, list):
        return True
    return isinstance(v, dict) and any(_has_list(x) for x in v.values())


def test_batch_equals_per_record_on_goldens():
    got, counts = _check([json.loads(json.dumps(c["values"])) for c in load_golden("alignment")])
    assert all(g is not None for g in got) and counts["device_pairs"] > 0


def test_batch_equals_per_record_on_random_structures():
    from oracle.gen_golden import _record_candidates
    rng = random.Random(20261015)
    records = random_records(rng, 4000)
    for n in (2, 3, 5, 8, 16, 32):
        records += [json.loads(json.dumps(_record_candidates(rng, n, depth=3))) for _ in range(1000)]
    got, counts = _check(records)
    # the records hold nodes of > 512 elements, lists inside list elements and lists with two long strings (the last need the
    # Python pre-pass: None)
    long_pair = [i for i, r in enumerate(records[:4000]) if any("a" * 60 in json.dumps(v) for v in r)]
    assert long_pair and any(got[i] is None for i in long_pair)
    assert counts["device_pairs"] > 0 and counts["host_pairs"] > 0


def test_config3_pairs_are_decided_on_the_device():
    rng = random.Random(3)
    records = _config3(rng, 2000)
    got, counts = _check(records)
    assert sum(g is not None for g in got) == len(records)
    assert counts["device_pairs"] > 0 and counts["host_pairs"] == 0, counts  # lists of scalars: every pair is the device's


def test_consolidation_of_config3_texts_equals_host_logic():
    from k_llms_b200 import _native as K
    rng = random.Random(33)
    texts = [[json.dumps(c) for c in rec] for rec in _config3(rng, 3000)]
    exp = consolidate_json_with_oracle(texts)
    assert sum(e is not None for e in exp) > 2000
    assert K.consolidate_json(texts) == exp
    blob, off, n = K.pack_texts(texts)
    res = K.consolidate_json_packed(blob, off, n)
    try:
        for r, t in enumerate(texts):
            assert (res.status[r] == 1) == (exp[r] is None), (r, res.status[r])
            if exp[r] is not None:
                assert (res.content(r), res.likelihoods(r)) == exp[r], t
            if any(_has_list(json.loads(x)) for x in t):
                assert res.status[r] != 0  # the device JSON path still declines records with list fields
    finally:
        res.close()
