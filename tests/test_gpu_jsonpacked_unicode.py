"""GPU parity for KC_JSON_UNICODE on the device JSON path: similarity-medoid fields with non-ASCII text or \\uXXXX escapes.  The
kernels must give what the host instantiation of the same phases gives (tests/test_jsongpu_unicode_host_logic.py pins that to the
reference's goldens), byte for byte, for the count and weighted entry points; the client functions must answer such records
on the device with the Python route's value and likelihoods.  Nothing here needs Unidecode: vote fields stay ASCII."""
import asyncio
import json

import numpy as np
import pytest

from k_llms_b200 import _native as K
from tests.helpers import jsongpu_with_oracle, load_golden
from tools.gen_golden_unicode import unicode_records

pytestmark = pytest.mark.gpu
UNI = K.JSON_UNICODE | K.JSON_KEY_UNION | K.JSON_LISTS


def _records():
    by_n = {}
    for case in load_golden("unicode_medoid"):
        by_n.setdefault(len(case["texts"]), []).append((case["texts"], (case["content"], case["likelihoods"])))
    for texts in unicode_records(77, 600, ns=(2, 3, 5, 8, 16, 33, 64), reshape=True):
        by_n.setdefault(len(texts), []).append((texts, None))
    return by_n


def _device(recs, seq=None, flags=UNI):
    blob, off, n = K.pack_texts(recs)
    if seq is None:
        res = K.consolidate_json_packed(blob, off, n, flags=flags | K.JSON_DEVICE_ONLY)
    else:
        res = K.consolidate_json_packed_weighted(blob, off, n, seq, flags=flags)
    try:
        return res.pairs(), res.stats.n_device
    finally:
        res.close()


@pytest.mark.parametrize("weighted", [False, True], ids=["count", "weighted"])
def test_device_equals_twin_and_goldens(weighted):
    rng = np.random.default_rng(3)
    on_device = 0
    for n, items in _records().items():
        recs = [t for t, _ in items]
        seq = (-rng.exponential(4.0, len(recs) * n)).astype(np.float32) if weighted else None
        twin, status = jsongpu_with_oracle(recs, seq, flags=UNI)
        got, n_dev = _device(recs, seq)
        for (texts, gold), g, t, st in zip(items, got, twin, status):
            assert g == t, (texts, g, t, st)
            if gold is not None and not weighted:
                assert st == 0 and g == gold, texts
        on_device += n_dev
    assert on_device > 500, on_device


def test_numeric_medoid_equals_twin():
    for _n, items in _records().items():
        recs = [t for t, _ in items]
        twin, _ = jsongpu_with_oracle(recs, flags=UNI | K.JSON_NUMERIC_MEDOID)
        got, _ = _device(recs, flags=UNI | K.JSON_NUMERIC_MEDOID)
        assert got == twin


async def _raising(texts):
    raise RuntimeError("no network in tests")


def _client_records():
    from tools.jsonpacked_throughput import invoice_texts
    return [t for t, gold in _records().get(3, []) if gold is not None][:40] + invoice_texts(40, 3, 5, accents=True)


@pytest.mark.parametrize("weighted", [False, True])
def test_clients_answer_on_the_device_like_the_python_route(weighted, monkeypatch):
    """The async functions (count and weighted), the weighted sync client and the batch API on records with non-ASCII medoid
    fields: the native route answers every one (the Python route is never asked) with the Python route's answer."""
    import random

    from openai.types.chat import ParsedChatCompletion

    from k_llms_b200.utils import consensus_utils as CU
    from k_llms_b200.utils import consolidation as C
    from tests.test_async_native_host_logic import _completion
    rng = random.Random(7 + weighted)
    embed = lambda t: [[0.0] for _ in t]  # noqa: E731  (never called: no pair of long strings)
    kw = {"vote_weighting": "likelihood"} if weighted else {}
    python_async, python_sync = C._consensus_async, C._consensus_of_choices_python
    asked = []
    monkeypatch.setattr(C, "_consensus_async", lambda *a, **k: asked.append("async") or python_async(*a, **k))
    monkeypatch.setattr(C, "_consensus_of_choices_python", lambda *a, **k: asked.append("sync") or python_sync(*a, **k))
    records = _client_records()
    lps_all = []
    for texts in records:
        lps = [[-rng.random() * 4, -rng.random()] for _ in texts] if weighted else None
        lps_all.append(lps)
        comp = _completion(texts, lps)
        contents = [json.loads(t) for t in texts]
        sums = C._sequence_logprobs(lps) if weighted else None
        out = asyncio.run(C.async_consolidate_parsed_chat_completions(ParsedChatCompletion.model_validate(comp.model_dump()), _raising,
                                                                      None, **kw))
        assert not asked, texts
        value, conf = asyncio.run(python_async(contents, CU.ConsensusSettings(), _raising, None, sums))
        assert out.choices[0].message.content == C._format_consensus_content(value) and out.likelihoods == conf, texts
        out = C.consolidate_chat_completions(comp, embed, None, **kw)
        assert not asked, texts
        value, conf = C._consensus_sync(contents, CU.ConsensusSettings(), embed, None, sums)
        assert out.choices[0].message.content == C._format_consensus_content(value) and out.likelihoods == conf, texts
    counts = {}
    batch = C.consolidate_contents_batch(records, get_openai_embeddings_from_text=embed, token_logprobs=lps_all if weighted else None,
                                         counts=counts)
    assert not asked
    if weighted:
        assert counts["device"] == len(records), counts
    for texts, lps, got in zip(records, lps_all, batch):
        sums = C._sequence_logprobs(lps) if weighted else None
        value, conf = C._consensus_sync([json.loads(t) for t in texts], CU.ConsensusSettings(), embed, None, sums)
        assert tuple(got) == (C._format_consensus_content(value), conf), texts
