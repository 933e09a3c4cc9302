"""GPU: the async dispatcher on the device — K5 (kc_numeric_medoid_f64) against its numpy oracle bit for bit, the device JSON path with
KC_JSON_NUMERIC_MEDOID against the reference's goldens and against its own phases run on the host, and the async entry points
against the Python async route."""
import asyncio
import json
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from k_llms_b200.utils import consensus_utils as CU
from k_llms_b200.utils import consolidation as C
from oracle import columnar as OC
from tests.async_native_oracle import cells_of, golden_cases, numeric_medoid
from tests.helpers import jsongpu_with_oracle
from tests.test_async_native_host_logic import _completion, random_numeric_groups

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


async def _raising(texts):
    raise RuntimeError("no network in tests")


def _k5(cells):
    best, avg = K.numeric_medoid(torch.from_numpy(np.ascontiguousarray(cells)).cuda())
    torch.cuda.synchronize()
    return best.cpu().numpy(), avg.cpu().numpy()


def _same(cells):
    best, avg = _k5(cells)
    eb, ea = numeric_medoid(cells)
    bad = np.flatnonzero((best != eb) | (avg.view(np.uint64) != ea.view(np.uint64)))
    assert bad.size == 0, (cells[bad[0]], best[bad[0]], avg[bad[0]], eb[bad[0]], ea[bad[0]])


@pytest.mark.parametrize("n", range(1, 65))
def test_k5_matches_oracle(n):
    rng = random.Random(n)
    G = 20_000 + rng.randrange(0, 97)  # ragged group counts: the last warp is partly idle
    _, cells = random_numeric_groups(rng, G, n)
    _same(cells)


def test_k5_agreeing_and_all_none_groups():
    for n in (2, 7, 16, 33, 64):
        cells = np.full((3000, n), 42.0)
        cells[1000:2000] = OC.F64_NONE
        cells[2000:, ::2] = OC.F64_ABSENT
        _same(cells)


def test_k5_on_reference_goldens():
    cases = golden_cases("group")
    by_n = {}
    for case in cases:
        by_n.setdefault(len(case["values"]), []).append(case)
    for n, group in by_n.items():
        cells = cells_of([c["values"] for c in group], n)
        best, avg = _k5(cells)
        for case, b, a in zip(group, best, avg):
            live = [v for v in case["values"] if v is not None]
            assert json.dumps(live[b]) == json.dumps(case["value"]), case
            conf = 1.0 * (len(live) / n) * 1.0 if len(live) == 1 else round(1.0 * (len(live) / n) * float(a), 5)
            assert conf == case["conf"], case


def _packed(records, seq=None, chunk_mb=None, monkeypatch=None):
    if chunk_mb is not None:
        monkeypatch.setenv("KC_JSON_CHUNK_MB", str(chunk_mb))
    blob, off, n = K.pack_texts(records)
    if seq is None:
        res = K.consolidate_json_packed(blob, off, n, flags=K.JSON_NUMERIC_MEDOID)
    else:
        res = K.consolidate_json_packed_weighted(blob, off, n, seq, flags=K.JSON_NUMERIC_MEDOID)
    try:
        return res.pairs(), list(res.status), list(res.why)
    finally:
        res.close()


def test_golden_texts_through_the_device_path():
    cases = golden_cases("texts")
    accepted = 0
    for case in cases:
        (got,), _, _ = _packed([case["texts"]])
        if got is not None:
            accepted += 1
            assert got == (case["content"], case["likelihoods"]), case
    assert accepted >= 30


def _fuzz_records(n, count, seed):
    from tests.test_json_fuzz import _records
    return _records(count, seed, ns=(n,))[n]


@pytest.mark.parametrize("n", [2, 3, 5, 8, 16, 33, 64])
@pytest.mark.parametrize("weighted", [False, True])
def test_device_path_matches_its_host_phases(n, weighted, monkeypatch):
    recs = _fuzz_records(n, 300, 777 + n)
    seq = (-np.random.default_rng(n).exponential(3.0, len(recs) * n)).astype(np.float32) if weighted else None
    exp_pairs, exp_status = jsongpu_with_oracle(recs, seq, flags=K.JSON_NUMERIC_MEDOID)
    for chunk_mb in (None, 1):
        pairs, status, why = _packed(recs, seq, chunk_mb, monkeypatch)
        assert [s != 0 for s in status] == [s != 0 for s in exp_status]
        assert [w for w in why] == [int(s) for s in exp_status]
        assert pairs == exp_pairs
    assert sum(p is not None for p in exp_pairs) > 30


def _records_for_clients(rng, count, n):
    out = []
    for r in range(count):
        kind = r % 3
        cands = []
        for _ in range(n):
            d = {"v": rng.choice([10, 10, 20, 20.0, 30, None]), "w": rng.choice([1.5, 1.51, 3.0]), "s": rng.choice(["a", "b"])}
            if kind == 1:
                d["inner"] = {"m": rng.choice([7, 7.0, 8]), "t": rng.choice([True, False])}
            if kind == 2:
                d["items"] = [rng.choice([1, 2]) for _ in range(rng.randrange(1, 3))]  # a list: the Python async route
            cands.append(json.dumps(d))
        out.append(cands)
    return out


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("parsed", [False, True])
def test_async_functions_match_the_python_async_route(weighted, parsed):
    from openai.types.chat import ParsedChatCompletion
    rng = random.Random(5 + weighted + 2 * parsed)
    for texts in _records_for_clients(rng, 60, rng.choice([2, 3, 5, 8])):
        lps = [[-rng.random() * 4, -rng.random()] for _ in texts] if weighted else None
        completion = _completion(texts, lps)
        kw = {"vote_weighting": "likelihood"} if weighted else {}
        if parsed:
            out = asyncio.run(C.async_consolidate_parsed_chat_completions(ParsedChatCompletion.model_validate(completion.model_dump()),
                                                                          _raising, None, **kw))
        else:
            out = asyncio.run(C.async_consolidate_chat_completions(completion, _raising, None, **kw))
        contents = [json.loads(t) for t in texts]
        sums = C._sequence_logprobs(lps) if weighted else None
        value, conf = asyncio.run(C._consensus_async(contents, CU.ConsensusSettings(), _raising, None, sums))
        assert out.choices[0].message.content == C._format_consensus_content(value), texts
        assert out.likelihoods == conf, texts


def test_concurrent_requests_are_combined(monkeypatch):
    rng = random.Random(99)
    records = [r for i, r in enumerate(_records_for_clients(rng, 384, 3)) if i % 3 != 2]  # device-path records only
    assert len(records) == 256
    seq_out = [asyncio.run(C.async_consolidate_chat_completions(_completion(t), _raising, None)) for t in records]
    calls = []
    real = C._native_consolidate

    def counting(recs, *a, **k):
        calls.append(len(recs))
        return real(recs, *a, **k)
    monkeypatch.setattr(C, "_native_consolidate", counting)

    async def main():
        return await asyncio.gather(*(C.async_consolidate_chat_completions(_completion(t), _raising, None) for t in records))
    outs = asyncio.run(main())
    assert sum(calls) == len(records) and len(calls) < len(records), calls
    for a, b in zip(outs, seq_out):
        assert a.choices[0].message.content == b.choices[0].message.content and a.likelihoods == b.likelihoods
