"""GPU parity for H1g (kc_consolidate_json_packed): candidate texts in -> consensus / likelihoods texts out with the JSON work on
the device, byte-identical to the reference's client order (json.loads -> align -> consensus -> json.dumps, restated by the
object-level oracle).  The same generators as tests/test_jsongpu_host_logic.py, where the oracle sits in K1 / K2's place."""
import json
import os
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from tests.helpers import general_and_mutated_records
from tests.test_gpu_json import _expected, _expected_with_lists
from tests.test_jsongpu_host_logic import _flat_record, _phrase_record, _shaped_record, s32_texts

pytestmark = pytest.mark.gpu


def run(records, flags=0):
    blob, off, n = K.pack_texts(records)
    res = K.consolidate_json_packed(blob, off, n, flags=flags)
    return res


def test_s32_records_on_the_device():
    for n in (2, 3, 5, 16, 33, 64):
        recs = s32_texts(200 if n <= 16 else 40, n, 100 + n)
        res = run(recs)
        assert not res.status.any(), (n, list(res.status), list(res.why))
        assert res.stats.n_device == len(recs)
        for r, texts in enumerate(recs):
            assert (res.content(r), res.likelihoods(r)) == _expected(texts), texts


def test_flat_records_device_and_host_share():
    rng = random.Random(3)
    by_n = {}
    for _ in range(1500):
        n = rng.choice([2, 3, 4, 5, 8, 16, 20, 40])
        by_n.setdefault(n, []).append(_flat_record(rng, n))
    on_device = 0
    for _n, recs in by_n.items():
        res = run(recs)
        for r, texts in enumerate(recs):
            if res.status[r] == 1:
                continue
            on_device += res.status[r] == 0
            assert (res.content(r), res.likelihoods(r)) == _expected(texts), (texts, res.status[r], res.why[r])
    assert on_device > 1200


def test_phrase_fields_medoid_on_the_device():
    """Multi-word string fields: A2 builds K4's CSR input on the device, K4 picks the medoid, C0 / C1 print the winner's original
    text — byte-identical to the reference's client order."""
    rng = random.Random(29)
    by_n = {}
    for _ in range(1500):
        n = rng.choice([2, 3, 4, 5, 8, 16, 33])
        by_n.setdefault(n, []).append(_phrase_record(rng, n))
    on_device = 0
    for _n, recs in by_n.items():
        res = run(recs)
        for r, texts in enumerate(recs):
            if res.status[r] == 1:
                continue
            on_device += res.status[r] == 0
            assert (res.content(r), res.likelihoods(r)) == _expected(texts), (texts, res.status[r], res.why[r])
    assert on_device > 1200
    # many records, several chunks: the CSR offsets stay consistent across records declined at different stages
    recs = [_phrase_record(rng, 8) for _ in range(6000)]
    recs[17] = ['{"a": "the big cat", "b": 1e999}'] * 8          # declined while encoding, after its medoid group was counted
    res = run(recs)
    assert res.stats.n_device > 5000
    for r in random.Random(5).sample(range(len(recs)), 400) + [16, 17, 18]:
        if res.status[r] != 1:
            assert (res.content(r), res.likelihoods(r)) == _expected_with_lists(recs[r]), (recs[r], res.status[r])


def test_nested_objects_on_the_device():
    """Candidates of one shape with nested objects (depth <= 4): structure tokens, per-level key order and the nested output are
    the device's; byte-identical to the reference's client order."""
    rng = random.Random(41)
    by_n = {}
    for _ in range(1500):
        n = rng.choice([2, 3, 4, 5, 8, 16, 33])
        by_n.setdefault(n, []).append(_shaped_record(rng, n))
    on_device = nested = 0
    for _n, recs in by_n.items():
        res = run(recs)
        for r, texts in enumerate(recs):
            if res.status[r] == 1:
                continue
            if res.status[r] == 0:
                on_device += 1
                nested += any(isinstance(v, dict) for v in json.loads(texts[0]).values())
            assert (res.content(r), res.likelihoods(r)) == _expected(texts), (texts, res.status[r], res.why[r])
    assert on_device > 1300 and nested > 700, (on_device, nested)


def test_general_and_mutated_records_never_wrong():
    by_n = general_and_mutated_records(11)
    counts = {0: 0, 1: 0, 2: 0}
    for _n, recs in by_n.items():
        res = run(recs)
        for r, texts in enumerate(recs):
            counts[int(res.status[r])] += 1
            if res.status[r] != 1:
                assert (res.content(r), res.likelihoods(r)) == _expected_with_lists(texts), (texts, res.status[r])
    assert counts[0] > 200 and counts[2] > 200, counts


def test_device_only_flag_and_reasons():
    recs = [['{"a": "x\\u0041y"}', '{"a": "x"}'], ['{"a": 1, "b": "q"}', '{"a": 1, "b": "Q!"}'], ['{"a": [1]}', '{"a": [1]}'],
            ['{"a\x7f": "x y z"}', '{"a\x7f": "x y z"}']]  # DEL in a key: the host path prints it as \u007f
    res = run(recs, flags=K.JSON_DEVICE_ONLY)
    assert list(res.status) == [1, 0, 1, 1] and res.why[0] != 0 and res.why[2] != 0 and res.why[3] != 0
    assert res.content(1) == '{"a": 1.0, "b": "q"}' and res.likelihoods(1) == '{"a": 1.0, "b": 1.0}'
    res = run(recs)
    assert list(res.status) == [2, 0, 2, 2]
    for r, texts in enumerate(recs):
        assert (res.content(r), res.likelihoods(r)) == _expected_with_lists(texts)


def test_many_chunks_and_streams_agree_with_the_host_path(monkeypatch):
    """60k S32 records at n = 16 (~0.5 GB of JSON) cut into 8 MB chunks over 3 streams: every record equals what the HOST path
    (kc_consolidate_json, an independent implementation) produces, and a sample equals the oracle."""
    R, n = 60000, 16
    blob, off = K.s32_texts_packed(R, n, 4242)
    monkeypatch.setenv("KC_JSON_CHUNK_MB", "8")
    res = K.consolidate_json_packed(blob, off, n)
    assert not res.status.any() and res.stats.chunks > 30 and res.stats.n_device == R
    monkeypatch.setenv("KC_JSON_CHUNK_MB", "64")
    res1 = K.consolidate_json_packed(blob, off, n)
    text = blob.tobytes()
    sample = random.Random(1).sample(range(R), 150)
    for r in sample:
        texts = [text[off[r * n + c]:off[r * n + c + 1]].decode() for c in range(n)]
        assert (res.content(r), res.likelihoods(r)) == _expected(texts)
    for r in range(0, R, 7):
        assert res.content(r) == res1.content(r) and res.likelihoods(r) == res1.likelihoods(r)
    sub = 5000
    records = [[text[off[r * n + c]:off[r * n + c + 1]].decode() for c in range(n)] for r in range(sub)]
    host = K.consolidate_json(records)
    for r in range(sub):
        assert host[r] == (res.content(r), res.likelihoods(r)), r
