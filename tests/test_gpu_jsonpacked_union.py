"""GPU parity for the device JSON path's key-union round (U1-U3, k_llms_b200/csrc/kc_jsongpu.cuh): records whose candidates
reorder, lack or add keys, or hold None / nothing where others hold a sub-object, through kc_consolidate_json_packed with
JSON_KEY_UNION, its weighted variant, JSON_DEVICE_ONLY and JSON_NUMERIC_MEDOID, and through the client functions (which set the
flag).  Each result must equal the host instantiation of the same phases, the reference's client order and the host path; the
union records must stay on the device.  Without the flag the device declines them as its host instantiation does."""
import asyncio
import json
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from k_llms_b200.utils import consensus_utils as CU
from k_llms_b200.utils import consolidation as C
from tests.helpers import jsongpu_with_oracle
from tests.test_async_native_host_logic import _completion
from tests.test_gpu_json import _expected
from tests.test_jsongpu_host_logic import _shaped_record, s32_texts
from tests.test_jsongpu_union_host_logic import ACCEPTED, DECLINED, union_record, union_records

pytestmark = pytest.mark.gpu


def _run(records, flags=0, seq=None, key_union=True):
    blob, off, n = K.pack_texts(records)
    flags |= K.JSON_KEY_UNION if key_union else 0
    res = (K.consolidate_json_packed(blob, off, n, flags=flags) if seq is None else
           K.consolidate_json_packed_weighted(blob, off, n, seq, flags=flags))
    try:
        return res.pairs(), [int(s) for s in res.status], [int(w) for w in res.why], res.stats.as_dict()
    finally:
        res.close()


def test_union_records_count_vote():
    for n, recs in union_records(101, 1400).items():
        exp, exp_status = jsongpu_with_oracle(recs, flags=K.JSON_KEY_UNION)
        host = K.consolidate_json(recs)
        for flags in (0, K.JSON_DEVICE_ONLY):
            pairs, status, why, stats = _run(recs, flags)
            assert status == [0] * len(recs) and why == [int(s) for s in exp_status], n
            assert stats["n_device"] == len(recs) and stats["n_host"] == 0, stats
            assert pairs == exp, n
        for r, texts in enumerate(recs):
            assert pairs[r] == _expected(texts) == host[r], texts
        # without the flag: declined as before, exactly where the host instantiation without it declines
        old, old_status = jsongpu_with_oracle(recs)
        pairs, status, why, stats = _run(recs, K.JSON_DEVICE_ONLY, key_union=False)
        assert why == [int(s) for s in old_status] and pairs == old, n


def test_union_records_weighted_and_async_medoid():
    rng = np.random.default_rng(3)
    for n, recs in union_records(202, 600, ns=(2, 3, 5, 8, 16, 33, 64)).items():
        seq = (-rng.exponential(4.0, len(recs) * n)).astype(np.float32)
        exp, _ = jsongpu_with_oracle(recs, seq, flags=K.JSON_KEY_UNION)
        pairs, status, _, stats = _run(recs, seq=seq)
        assert status == [0] * len(recs) and stats["n_device"] == len(recs)
        assert pairs == exp, n
        for s in (None, seq):
            exp, exp_status = jsongpu_with_oracle(recs, s, flags=K.JSON_KEY_UNION | K.JSON_NUMERIC_MEDOID)
            pairs, status, why, stats = _run(recs, K.JSON_NUMERIC_MEDOID, s)
            assert why == [int(x) for x in exp_status] and not any(status) and stats["n_device"] == len(recs), n
            assert pairs == exp, n


def test_union_edges_on_the_device():
    for name, texts in ACCEPTED.items():
        (got,), (st,), _, _ = _run([texts], K.JSON_DEVICE_ONLY)
        assert st == 0 and got == _expected(texts), name
    for name, (texts, why) in DECLINED.items():
        (got,), (st,), (w,), _ = _run([texts], K.JSON_DEVICE_ONLY)
        assert got is None and st == 1 and w == why, (name, w)
        (got,), (st,), _, _ = _run([texts])  # the host path takes what it models
        assert (got is None) == (st == 1), name


def test_mixed_chunks(monkeypatch):
    """1 MB chunks: same-shape and union records interleaved, a run of chunks without union records, a run of chunks that
    are all union records; every record equals the 64 MB run and the host instantiation."""
    rng = random.Random(17)
    mixed = [union_record(rng, 8) if i % 2 else _shaped_record(rng, 8) for i in range(3000)]
    plain = s32_texts(4000, 8, 5)
    only = [union_record(rng, 8) for _ in range(3000)]
    recs = mixed + plain + only
    exp, exp_status = jsongpu_with_oracle(recs, flags=K.JSON_KEY_UNION)
    monkeypatch.setenv("KC_JSON_CHUNK_MB", "64")
    big = _run(recs, K.JSON_DEVICE_ONLY)
    monkeypatch.setenv("KC_JSON_CHUNK_MB", "1")
    small = _run(recs, K.JSON_DEVICE_ONLY)
    assert small[3]["chunks"] > 5 and big[3]["chunks"] == 1
    assert small[:3] == big[:3]
    assert small[0] == exp and small[2] == [int(s) for s in exp_status]
    for seed in (1, 2):
        monkeypatch.setenv("KC_JSON_STREAMS", str(seed))
        assert _run(recs, K.JSON_DEVICE_ONLY)[:3] == big[:3]


def _reordered_requests(rng, count, n):
    out = []
    for _ in range(count):
        cands = []
        for _c in range(n):
            items = [("v", rng.choice([10, 10, 20, 20.0, 30, None])), ("w", rng.choice([1.5, 1.51, 3.0])), ("s", rng.choice(["a", "b"]))]
            if rng.random() < 0.5:
                items.append(("inner", None if rng.random() < 0.3 else {"m": rng.choice([7, 7.0, 8]), "t": rng.choice([True, False])}))
            if rng.random() < 0.3:
                del items[rng.randrange(len(items))]
            rng.shuffle(items)
            cands.append(json.dumps(dict(items)))
        out.append(cands)
    return out


async def _raising(texts):
    raise RuntimeError("no network in tests")


@pytest.mark.parametrize("weighted", [False, True])
def test_clients_keep_reordered_requests_native(weighted, monkeypatch):
    """The async functions (and, weighted, the sync client) on requests whose candidates reorder or lack keys or hold None for a
    sub-object: the native route answers every one (the Python route is never asked) and equals the Python route's answer."""
    from openai.types.chat import ParsedChatCompletion
    rng = random.Random(41 + weighted)
    embed = lambda t: [[0.0] for _ in t]  # noqa: E731
    kw = {"vote_weighting": "likelihood"} if weighted else {}
    python_async, python_sync = C._consensus_async, C._consensus_of_choices_python
    asked = []
    monkeypatch.setattr(C, "_consensus_async", lambda *a, **k: asked.append("async") or python_async(*a, **k))
    monkeypatch.setattr(C, "_consensus_of_choices_python", lambda *a, **k: asked.append("sync") or python_sync(*a, **k))
    for texts in _reordered_requests(rng, 60, 5):
        lps = [[-rng.random() * 4, -rng.random()] for _ in texts] if weighted else None
        comp = _completion(texts, lps)
        contents = [json.loads(t) for t in texts]
        sums = C._sequence_logprobs(lps) if weighted else None
        out = asyncio.run(C.async_consolidate_parsed_chat_completions(ParsedChatCompletion.model_validate(comp.model_dump()), _raising,
                                                                      None, **kw))
        assert not asked, texts
        value, conf = asyncio.run(python_async(contents, CU.ConsensusSettings(), _raising, None, sums))
        assert out.choices[0].message.content == C._format_consensus_content(value) and out.likelihoods == conf, texts
        if weighted:
            out = C.consolidate_chat_completions(comp, embed, None, **kw)
            assert not asked, texts
            value, conf = C._consensus_sync(contents, CU.ConsensusSettings(), embed, None, sums)
            assert out.choices[0].message.content == C._format_consensus_content(value) and out.likelihoods == conf, texts
