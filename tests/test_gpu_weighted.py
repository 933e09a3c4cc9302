"""GPU: likelihood-weighted consensus (DESIGN.md §5) — K3b over ragged records (kc_weighted_vote_groups_i8) against the C
oracle bit for bit, and the product entry points against the weighted oracle."""
import asyncio
import json

import numpy as np
import pytest

from oracle import columnar as OC
from oracle import consensus_py as O
from tests import weighted_oracle as W
from tests.helpers import jsongpu_with_oracle, same
from tests.test_weighted_host_logic import _completion, _flat_records, _seq, _wrapped, random_record

pytestmark = pytest.mark.gpu
EMBED = lambda texts: [[0.0] for _ in texts]  # noqa: E731


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _ragged_case(rng, n, G, R):
    codes = rng.integers(0, max(1, min(n, 6)), (G, n)).astype(np.int8)
    codes[rng.random((G, n)) < 0.1] = -1
    codes[rng.random((G, n)) < 0.05] = -2
    kind = rng.integers(0, 4, R)
    seq = np.where(kind[:, None] == 0, np.float32(-2.0),
          np.where(kind[:, None] == 1, -rng.exponential(3.0, (R, n)),
          np.where(kind[:, None] == 2, rng.choice([-9999.0, -0.25], (R, n)), -rng.integers(0, 3, (R, n)) * np.log(3.0)))).astype(np.float32)
    # shuffled, non-monotonic record indices; every fifth record has no group at all
    with_groups = np.array([r for r in range(R) if r % 5 != 3], dtype=np.int32)
    rec = with_groups[rng.integers(0, len(with_groups), G)].astype(np.int32)
    return codes, rec, seq


def _run(torch, codes, rec, seq):
    from k_llms_b200 import _native as K
    win, meta, weight = K.weighted_vote_groups(torch.from_numpy(codes).cuda(), torch.from_numpy(rec).cuda(), torch.from_numpy(seq).cuda())
    torch.cuda.synchronize()
    return win.cpu().numpy(), meta.cpu().numpy().view(np.uint32), weight.cpu().numpy()


def _check(got, codes, rec, seq):
    ew, em, ewt = OC.weighted_vote(codes.astype(np.int32)[:, None, :], seq[rec])
    assert np.array_equal(got[0], ew)
    assert np.array_equal(got[1], em)
    assert np.array_equal(got[2].view(np.uint32), ewt.view(np.uint32))


@pytest.mark.parametrize("n", list(range(1, 65)))
def test_groups_kernel_matches_oracle(n):
    torch = _torch()
    rng = np.random.default_rng(9000 + n)
    G = 2000 + 37 * n  # not a multiple of the block size
    codes, rec, seq = _ragged_case(rng, n, G, R=max(1, G // 7))
    _check(_run(torch, codes, rec, seq), codes, rec, seq)


@pytest.mark.parametrize("n", [3, 16, 32, 64])
def test_groups_kernel_several_waves(n):
    torch = _torch()
    rng = np.random.default_rng(77 + n)
    G = 400_003  # several waves of the grid-stride loop
    codes, rec, seq = _ragged_case(rng, n, G, R=G // 24 + 1)
    _check(_run(torch, codes, rec, seq), codes, rec, seq)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 12, 16, 24, 32, 48, 64])
@pytest.mark.parametrize("F", [1, 5, 24])
def test_groups_kernel_equals_fixed_shape_k3b(n, F):
    """group_record[g] = g / F: the same result as kc_weighted_vote_i32 on the same cells (every path it dispatches to)."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(n * 100 + F)
    R = 3001
    codes, _, seq = _ragged_case(rng, n, R * F, R)
    rec = (np.arange(R * F) // F).astype(np.int32)
    got = _run(torch, codes, rec, seq)
    w, m, wt = K.weighted_vote(torch.from_numpy(codes.astype(np.int32).reshape(R, F, n)).cuda(), torch.from_numpy(seq).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(got[0], w.cpu().numpy())
    assert np.array_equal(got[1], m.cpu().numpy().view(np.uint32))
    assert np.array_equal(got[2].view(np.uint32), wt.cpu().numpy().view(np.uint32))


def test_contents_batch_weighted_matches_oracle():
    _torch()
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from k_llms_b200.utils.consolidation import _aligned_sync, _format_consensus_content, _safe_parse_content, consolidate_contents_batch
    rng = np.random.default_rng(2026)
    records, lps = [], []
    for i in range(3000):
        n = int(rng.choice([2, 3, 5, 8, 16, 32]))
        if i % 2:
            records.append([json.dumps(c) if rng.random() > 0.05 else "" for c in random_record(rng, n)])
        else:  # flat records of one key sequence: the device path's ground
            records.append(_flat_records(rng, 1, n)[0])
        lps.append([list(-rng.exponential(0.7, int(rng.integers(0, 40)))) for _ in range(n)])
    counts = {}
    got = consolidate_contents_batch(records, token_logprobs=lps, counts=counts)
    for texts, toks, g in zip(records, lps, got):
        keep = [c for c, t in enumerate(texts) if t]
        flat = np.asarray([x for c in keep for x in toks[c]], dtype=np.float32)
        off = np.asarray([0] + list(np.cumsum([len(toks[c]) for c in keep])), dtype=np.int64)
        seq = OC.logprob_sum(flat, off)
        contents = [_safe_parse_content(texts[c]) for c in keep]
        aligned = _aligned_sync(contents, ConsensusSettings(), EMBED, None)
        value, conf = W.client_order(contents, seq, O.DEFAULTS, EMBED, aligned=aligned)
        assert g[0] == _format_consensus_content(value) and same(g[1], conf), (texts, g, value, conf)
    print(f"\n{len(records)} records consolidated with likelihood-weighted votes, {counts['device']} of them on the device JSON path")
    assert counts["device"] >= 1000


def test_four_consolidation_functions_and_client():
    _torch()
    from openai.types.chat import ParsedChatCompletion
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from k_llms_b200.utils.consolidation import (_aligned_sync, async_consolidate_chat_completions, async_consolidate_parsed_chat_completions,
                                                 consolidate_chat_completions, consolidate_parsed_chat_completions)
    rng = np.random.default_rng(31)
    for i in range(60):
        n = int(rng.choice([2, 3, 5, 8]))
        if i % 2:  # flat records: the weighted device JSON path through the per-request combiner
            cands = [json.loads(t) for t in _flat_records(rng, 1, n)[0]]
        else:
            cands = [c if isinstance(c, dict) else {"text": c} for c in random_record(rng, n)]
        texts = [json.dumps(c) for c in cands]
        toks = [list(-rng.exponential(0.5, int(rng.integers(1, 12)))) for _ in range(n)]
        comp = _completion(texts, toks)
        seq = OC.logprob_sum(np.asarray([x for t in toks for x in t], dtype=np.float32),
                             np.asarray([0] + list(np.cumsum([len(t) for t in toks])), dtype=np.int64))
        aligned = _aligned_sync(cands, ConsensusSettings(), EMBED, None)
        exp = W.client_order(cands, seq, O.DEFAULTS, EMBED, aligned=aligned)
        out = consolidate_chat_completions(comp, EMBED, None, vote_weighting="likelihood")
        assert (json.loads(out.choices[0].message.content), out.likelihoods) == exp
        pc = ParsedChatCompletion.model_validate(comp.model_dump())
        out = consolidate_parsed_chat_completions(pc, EMBED, None, vote_weighting="likelihood")
        assert (json.loads(out.choices[0].message.content), out.likelihoods) == exp

        async def aembed(texts):
            return EMBED(texts)
        a1 = asyncio.run(async_consolidate_chat_completions(comp, aembed, None, vote_weighting="likelihood"))
        a2 = asyncio.run(async_consolidate_parsed_chat_completions(pc, aembed, None, vote_weighting="likelihood"))
        for a in (a1, a2):
            got = json.loads(a.choices[0].message.content)
            # vote leaves are weighted the same way in the async twin (values and likelihoods); numbers take the async
            # dispatcher's medoid
            for k in ("status", "flag", "addr"):
                assert got.get(k) == exp[0].get(k) and a.likelihoods.get(k) == exp[1].get(k), (k, got, a.likelihoods, exp)
        for method in ("create", "parse"):
            w, rec = _wrapped(False, comp)
            kw = dict(messages=[{"role": "user", "content": "q"}], model="m", n=n)
            if method == "parse":
                kw["response_format"] = None
            out = getattr(w.chat.completions, method)(**kw, vote_weighting="likelihood")
            assert rec.calls[-1]["logprobs"] is True
            assert (json.loads(out.choices[0].message.content), out.likelihoods) == exp


@pytest.mark.parametrize("n", [2, 3, 5, 8, 16, 32])
def test_weighted_device_json_path_matches_host_phases(n):
    """kc_consolidate_json_packed_weighted on the GPU against its phases on the host with the C oracle in the kernels' place:
    the same texts byte for byte, the same declined records."""
    _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(700 + n)
    records = _flat_records(rng, 2000, n)
    seq = np.concatenate([_seq(rng, n) for _ in records]).astype(np.float32)
    exp, status = jsongpu_with_oracle(records, seq)
    blob, off, _ = K.pack_texts(records)
    res = K.consolidate_json_packed_weighted(blob, off, n, seq)
    try:
        got = res.pairs()
        assert [p is None for p in got] == [s != 0 for s in status]  # declined records keep status 1: no host path
        assert got == exp
        assert res.stats.n_device == sum(p is not None for p in exp) > 1000 and res.stats.n_host == 0
    finally:
        res.close()
