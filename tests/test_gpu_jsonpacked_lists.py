"""GPU parity for the device JSON path's list round (KC_JSON_LISTS, k_llms_b200/csrc/kc_jsongpu.cuh): records with list fields
through kc_consolidate_json_packed, its weighted variant and JSON_NUMERIC_MEDOID, and through the client functions (which set the
flag).  Each result must equal the host instantiation of the same phases byte for byte, and the list records must come back from
the device (status 0).  Chunk size and stream count change nothing."""
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
from tests.test_jsongpu_host_logic import s32_texts
from tests.test_jsongpu_lists_host_logic import LISTS, list_records
from tests.test_jsongpu_union_host_logic import union_record
from tools.jsonpacked_throughput import invoice_lines_texts

pytestmark = pytest.mark.gpu


def _run(records, flags=0, seq=None):
    blob, off, n = K.pack_texts(records)
    flags |= LISTS
    res = (K.consolidate_json_packed(blob, off, n, flags=flags) if seq is None else
           K.consolidate_json_packed_weighted(blob, off, n, seq, flags=flags))
    try:
        return res.pairs(), [int(s) for s in res.status], [int(w) for w in res.why], res.stats.as_dict()
    finally:
        res.close()


def test_list_records_equal_the_host_instantiation():
    rng = np.random.default_rng(5)
    on_device = 0
    for n, recs in list_records(71, 1200).items():
        count, count_status = jsongpu_with_oracle(recs, flags=LISTS)
        pairs, status, why, stats = _run(recs, K.JSON_DEVICE_ONLY)
        assert why == count_status and pairs == count, n
        assert status == [1 if s else 0 for s in count_status] and stats["n_device"] == count_status.count(0), stats
        on_device += stats["n_device"]
        seq = (-rng.exponential(4.0, len(recs) * n)).astype(np.float32)
        exp, exp_status = jsongpu_with_oracle(recs, seq, flags=LISTS)
        pairs, status, why, stats = _run(recs, seq=seq)
        assert why == exp_status and pairs == exp, n
        exp, exp_status = jsongpu_with_oracle(recs, flags=LISTS | K.JSON_NUMERIC_MEDOID)
        pairs, status, why, stats = _run(recs, K.JSON_NUMERIC_MEDOID)
        assert why == exp_status and pairs == exp, n
        # the sync count vote hands what the device declines to the host path, with the original texts
        pairs, status, _, _ = _run(recs)
        host = K.consolidate_json(recs)
        for r, st in enumerate(status):
            assert pairs[r] == (count[r] if st == 0 else host[r]) and (st == 0) == (count_status[r] == 0), recs[r]
    assert on_device > 1000, on_device


def test_invoice_lines_on_the_device():
    recs = invoice_lines_texts(2000, 16, 3)
    exp, exp_status = jsongpu_with_oracle(recs, flags=LISTS)
    pairs, status, why, stats = _run(recs)
    assert pairs == exp and status == [0] * len(recs) and stats["n_device"] == len(recs) and stats["n_host"] == 0, stats


def test_mixed_chunks_and_streams(monkeypatch):
    """1 MB chunks and 1-3 streams, list and non-list records interleaved: every record equals the 64 MB run and the host
    instantiation."""
    rng = random.Random(19)
    lists = invoice_lines_texts(3000, 8, 7)
    plain = s32_texts(3000, 8, 5)
    recs = []
    for i in range(3000):
        recs += [lists[i], plain[i], union_record(rng, 8)]
    exp, exp_status = jsongpu_with_oracle(recs, flags=LISTS)
    monkeypatch.setenv("KC_JSON_CHUNK_MB", "64")
    big = _run(recs, K.JSON_DEVICE_ONLY)
    assert big[0] == exp and big[2] == exp_status
    monkeypatch.setenv("KC_JSON_CHUNK_MB", "1")
    for streams in ("1", "2", "3"):
        monkeypatch.setenv("KC_JSON_STREAMS", streams)
        small = _run(recs, K.JSON_DEVICE_ONLY)
        assert small[3]["chunks"] > 5 and small[:3] == big[:3], streams


def _list_requests(rng, count, n):
    out = []
    for _ in range(count):
        truth = [{"sku": rng.choice(["A1", "B2", "C3"]), "qty": rng.choice([1, 2, 3]), "price": rng.choice([1.5, 2.0, 9.99])}
                 for _ in range(rng.randrange(1, 5))]
        cands = []
        for _c in range(n):
            items = [dict(t, qty=t["qty"] + (rng.random() < 0.2)) for t in truth]
            if len(items) > 1 and rng.random() < 0.3:
                del items[rng.randrange(len(items))]
            rng.shuffle(items)
            cands.append(json.dumps({"items": items, "tags": rng.sample(["x", "y", "z"], rng.randrange(1, 3)), "total": rng.choice([10, 10.5])}))
        out.append(cands)
    return out


async def _raising(texts):
    raise RuntimeError("no network in tests")


@pytest.mark.parametrize("weighted", [False, True])
def test_clients_keep_list_requests_native(weighted, monkeypatch):
    """The async functions (count and weighted) and the weighted sync client on requests with list fields: the native route
    answers every one (the Python route is never asked) and equals the Python route's answer."""
    from openai.types.chat import ParsedChatCompletion
    rng = random.Random(43 + weighted)
    embed = lambda t: [[0.0] for _ in t]  # noqa: E731
    kw = {"vote_weighting": "likelihood"} if weighted else {}
    python_async, python_sync = C._consensus_async, C._consensus_of_choices_python
    asked = []
    monkeypatch.setattr(C, "_consensus_async", lambda *a, **k: asked.append("async") or python_async(*a, **k))
    monkeypatch.setattr(C, "_consensus_of_choices_python", lambda *a, **k: asked.append("sync") or python_sync(*a, **k))
    for texts in _list_requests(rng, 60, 5):
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
