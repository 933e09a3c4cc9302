"""The async dispatcher on the device JSON path (KC_JSON_NUMERIC_MEDOID), checked on the CPU:
  - K5's oracle (numpy's nanmean / argmax over stacks of groups) against numpy's nanmean / argmax on each group's own matrix, as
    similarity.medoid builds it, and against the running reference's async_consensus_values (tests/golden/async_numeric.json, oracle/gen_golden_async_numeric.py);
  - the device phases under the flag, instantiated on the host with the oracle in the kernels' place, against the golden texts
    and the Python async route, byte for byte; numeric fields that also hold strings or bools are declined;
  - the async entry points take the native route when a device is there (the host phases standing in for it)."""
import asyncio
import json
import math
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from k_llms_b200 import columnar
from k_llms_b200.utils import consensus_utils as CU
from k_llms_b200.utils import consolidation as C
from oracle import columnar as OC
from tests.async_native_oracle import cells_of, golden_cases, numeric_medoid, oracle_native_consolidate
from tests.helpers import jsongpu_with_oracle, oracle_run


async def _raising(texts):
    raise RuntimeError("no network in tests")


def numpy_medoid(values):
    """similarity.medoid's index and mean for numbers: the reference's matrix, np.nanmean, np.argmax."""
    k = len(values)
    sims = np.zeros((k, k), dtype=float)
    for i in range(k):
        for j in range(i + 1, k):
            sims[i, j] = sims[j, i] = 1.0 if math.isclose(values[i], values[j], rel_tol=0.01) else 1e-8
        sims[i, i] = np.nan
    avg = np.nanmean(sims, axis=1)
    best = int(np.argmax(avg))
    return best, float(avg[best])


def random_numeric_groups(rng, G, n):
    """Groups of n cells: few classes (ties), 1 % edges, +-0 / subnormals, +-inf, NaN payloads, None / absent cells."""
    groups = []
    for _ in range(G):
        style = rng.randrange(6)
        if style == 0:
            pool = [float(rng.choice([1, 10, 100]) * m) for m in rng.sample([1, 2, 3, 5, 7], rng.randint(2, 5))]
        elif style == 1:
            b = rng.choice([100.0, 1.0, 2.5, 1e6])
            pool = [b, b * 1.01, b * 0.99, b + b / 100, b - b / 100, b * 1.0100000000000002]
        elif style == 2:
            pool = [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 1e-300]
        elif style == 3:
            pool = [math.inf, -math.inf, 1.0, 1e308, -1e308]
        elif style == 4:
            pool = [math.nan, 1.0, 1.005, np.frombuffer(np.uint64(0x7FF0000000000001).tobytes(), np.float64)[0]]
        else:
            pool = [rng.uniform(-1e3, 1e3) for _ in range(3)] + [rng.uniform(-1, 1)]
        row = []
        for _ in range(n):
            r = rng.random()
            row.append(None if r < 0.1 else ("absent" if r < 0.15 else rng.choice(pool)))
        groups.append(row)
    cells = np.empty((G, n), dtype=np.float64)
    for g, row in enumerate(groups):
        cells[g] = [OC.F64_NONE if v is None else (OC.F64_ABSENT if v == "absent" else v) for v in row]
    return groups, cells


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 9, 16, 17, 31, 32, 33, 63, 64])
def test_oracle_matches_numpy(n):
    rng = random.Random(1000 + n)
    G = 110_000 // 15 + 1  # >= 100,000 groups over the parametrisation
    groups, cells = random_numeric_groups(rng, G, n)
    best, avg = numeric_medoid(cells)
    for g, row in enumerate(groups):
        live = [v for v in row if v is not None and v != "absent"]
        if len(live) < 2:
            assert best[g] == (0 if live else -1) and math.isnan(avg[g])
            continue
        eb, ea = numpy_medoid(live)
        assert best[g] == eb and np.float64(ea).tobytes() == avg[g].tobytes(), (live, best[g], avg[g], eb, ea)


def test_oracle_matches_reference_goldens():
    cases = golden_cases("group")
    assert len(cases) > 300
    by_n = {}
    for case in cases:
        by_n.setdefault(len(case["values"]), []).append(case)
    for n, group in by_n.items():
        best, avg = numeric_medoid(cells_of([c["values"] for c in group], n))
        for case, b, a in zip(group, best, avg):
            live = [v for v in case["values"] if v is not None]
            assert json.dumps(live[b]) == json.dumps(case["value"]), case  # the same number, printed the same way
            conf = 1.0 * (len(live) / n) * 1.0 if len(live) == 1 else round(1.0 * (len(live) / n) * float(a), 5)
            assert conf == case["conf"], (case, a)


def test_count_first_is_not_the_rule():
    """Rows 0 and 2 of [10, 10, 20, 20, 30] have the same close-count; row 2 wins by one ulp (the reference says 20)."""
    best, avg = numeric_medoid(cells_of([[10, 10, 20, 20, 30], [10, 10, 20, 20]], 5))
    assert list(best) == [2, 2]
    assert round(avg[0], 5) == 0.25 and round(avg[1], 5) == 0.33333


def test_device_phases_match_golden_texts():
    cases = golden_cases("texts")
    assert len(cases) > 40
    accepted = 0
    for case in cases:
        (got,), (st,) = jsongpu_with_oracle([case["texts"]], flags=K.JSON_NUMERIC_MEDOID)
        if got is not None:
            accepted += 1
            assert got == (case["content"], case["likelihoods"]), (case, got)
    assert accepted >= 30, accepted  # the rest hold numbers outside the exact conversion range (1e-300, 20-digit ints): Python route


@pytest.fixture
def oracle_kernels(monkeypatch):
    monkeypatch.setattr(columnar.Plan, "run", lambda self, device=None: oracle_run(self))


def python_async(texts):
    """The Python async route's texts for one record (the oracle in the vote kernels' place)."""
    contents = [C._safe_parse_content(t) for t in texts if t]
    value, conf = asyncio.run(C._consensus_async(contents, CU.ConsensusSettings(), _raising, None))
    return C._format_consensus_content(value), json.dumps(conf)


def test_device_phases_match_python_async_route(oracle_kernels):
    from tests.test_json_fuzz import _records
    accepted = declined = 0
    for _n, recs in _records(1200, 4242, ns=(2, 3, 5, 8, 16)).items():
        pairs, status = jsongpu_with_oracle(recs, flags=K.JSON_NUMERIC_MEDOID)
        for texts, got, st in zip(recs, pairs, status):
            if got is None:
                declined += 1
                continue
            accepted += 1
            assert got == python_async(texts), (texts, st)
    assert accepted > 250 and declined > 0, (accepted, declined)


def test_mixed_numeric_fields_are_declined():
    records = [[json.dumps({"v": 0}), json.dumps({"v": False}), json.dumps({"v": 1})],
               [json.dumps({"v": 1}), json.dumps({"v": "1"}), json.dumps({"v": 1})],
               [json.dumps({"v": 1}), json.dumps({"v": None}), json.dumps({"v": 2})]]
    pairs, status = jsongpu_with_oracle(records, flags=K.JSON_NUMERIC_MEDOID)
    assert pairs[0] is None and pairs[1] is None and status[0] == status[1] == 11  # D_MIXED_TYPES
    assert pairs[2] is not None


def _completion(contents, logprobs=None):
    from openai.types.chat import ChatCompletion
    choices = []
    for i, c in enumerate(contents):
        ch = {"index": i, "finish_reason": "stop", "message": {"role": "assistant", "content": c}, "logprobs": None}
        if logprobs is not None:
            ch["logprobs"] = {"content": [{"token": "t", "logprob": x, "bytes": None, "top_logprobs": []} for x in logprobs[i]]}
        choices.append(ch)
    return ChatCompletion.model_validate({"id": "x", "object": "chat.completion", "created": 0, "model": "m", "choices": choices})


@pytest.fixture
def native_route(monkeypatch, oracle_kernels):
    """A device is 'there' and the device path's phases run on the host; records what reaches it."""
    import torch
    calls = []

    def consolidate(records, *a, **k):
        calls.append(len(records))
        return oracle_native_consolidate(records, *a, **k)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(C, "_native_consolidate", consolidate)
    monkeypatch.setattr(C, "_logprob_sums", lambda flat, off: OC.logprob_sum(flat, off))
    return calls


@pytest.mark.parametrize("parsed", [False, True])
def test_async_functions_take_the_native_route(native_route, parsed):
    texts = [json.dumps({"v": v, "s": s}) for v, s in ((10, "a"), (10, "a"), (20, "b"), (20, "b"))]
    completion = _completion(texts)
    if parsed:
        from openai.types.chat import ParsedChatCompletion
        completion = ParsedChatCompletion.model_validate(completion.model_dump())
        out = asyncio.run(C.async_consolidate_parsed_chat_completions(completion, _raising, None))
    else:
        out = asyncio.run(C.async_consolidate_chat_completions(completion, _raising, None))
    assert native_route == [1]
    assert json.loads(out.choices[0].message.content) == {"s": "a", "v": 20}
    assert out.likelihoods == {"s": 0.5, "v": 0.33333}
    assert out.choices[0].message.content == python_async(texts)[0]


def test_async_likelihood_weighting_takes_the_native_route(native_route, monkeypatch):
    from tests.test_weighted_host_logic import _oracle_run as weighted_oracle_run
    monkeypatch.setattr(columnar.Plan, "run", weighted_oracle_run)
    texts = [json.dumps({"v": v, "s": s}) for v, s in ((10, "a"), (10, "a"), (20, "b"), (20.0, "b"))]
    lps = [[-5.0], [-5.0], [-0.1], [-0.2]]
    out = asyncio.run(C.async_consolidate_chat_completions(_completion(texts, lps), _raising, None, vote_weighting="likelihood"))
    assert native_route == [1]
    assert json.loads(out.choices[0].message.content) == {"s": "b", "v": 20}  # the heavier class; the number's medoid as before
    contents = [json.loads(t) for t in texts]
    sums = C._sequence_logprobs(lps)
    value, conf = asyncio.run(C._consensus_async(contents, CU.ConsensusSettings(), _raising, None, sums))
    assert (out.choices[0].message.content, out.likelihoods) == (C._format_consensus_content(value), conf)


def test_declined_requests_take_the_python_async_route(native_route):
    texts = [json.dumps({"v": [1, 2]}), json.dumps({"v": [1, 2]}), json.dumps({"v": [1, 3]})]  # a list: not on the device path
    out = asyncio.run(C.async_consolidate_chat_completions(_completion(texts), _raising, None))
    assert native_route == [1]
    assert out.choices[0].message.content == python_async(texts)[0]


def test_concurrent_requests_share_device_calls(native_route):
    records = [[json.dumps({"v": i % 7, "w": (i * 3) % 5}), json.dumps({"v": i % 7, "w": 1}), json.dumps({"v": 2, "w": 1})] for i in range(64)]

    async def main():
        return await asyncio.gather(*(C.async_consolidate_chat_completions(_completion(t), _raising, None) for t in records))
    outs = asyncio.run(main())
    assert sum(native_route) == len(records) and len(native_route) < len(records)
    for t, out in zip(records, outs):
        assert out.choices[0].message.content == python_async(t)[0]


def test_without_a_device_the_async_route_is_unchanged(monkeypatch, oracle_kernels):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    monkeypatch.setattr(C, "_native_consolidate", lambda *a, **k: pytest.fail("the native route needs a device"))
    texts = [json.dumps({"v": 10}), json.dumps({"v": 10}), json.dumps({"v": 20}), json.dumps({"v": 20})]
    out = asyncio.run(C.async_consolidate_chat_completions(_completion(texts), _raising, None))
    assert json.loads(out.choices[0].message.content) == {"v": 20} and out.likelihoods == {"v": 0.33333}
