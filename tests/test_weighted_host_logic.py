"""CPU: likelihood-weighted consensus (DESIGN.md §5) without a GPU — the weighted oracle against a numpy restatement and
known answers, the weighted planner with the C oracle in the place of K3 / K3b, input checks, and the client keyword."""
import asyncio
import json
import math

import numpy as np
import pytest

from oracle import columnar as OC
from oracle import consensus_py as O
from tests import weighted_oracle as W
from tests.helpers import jsongpu_with_oracle, same

EMBED = lambda texts: [[0.0] for _ in texts]  # noqa: E731


# ----------------------------------------------------------------------------- the oracle itself

def _random_rows(rng, G, n):
    codes = rng.integers(0, max(1, min(n, 5)), (G, n)).astype(np.int32)
    codes[rng.random((G, n)) < 0.1] = -1
    codes[rng.random((G, n)) < 0.05] = -2
    kind = rng.integers(0, 4, G)
    seq = np.where(kind[:, None] == 0, np.float32(-1.5),                                  # equal sums: count-vote ties
          np.where(kind[:, None] == 1, -rng.exponential(3.0, (G, n)),
          np.where(kind[:, None] == 2, rng.choice([-9999.0, -0.5, -2.0], (G, n)),
                   -rng.integers(0, 3, (G, n)) * np.log(3.0)))).astype(np.float32)
    return codes, seq


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8, 13, 16, 31, 32, 33, 64])
def test_c_oracle_matches_numpy_restatement(n):
    rng = np.random.default_rng(100 + n)
    codes, seq = _random_rows(rng, 300, n)
    win, meta, weight = OC.weighted_vote(codes[:, None, :], seq)
    f = OC.meta_fields(meta)
    for g in range(len(codes)):
        code, first, share = W.brute_weighted_vote(codes[g], seq[g])
        assert int(win[g]) == code, (g, codes[g], seq[g])
        assert np.float32(weight[g]).view(np.uint32) == np.float32(share).view(np.uint32), (g, weight[g], share)
        if code >= 0:
            assert int(f["idx"][g]) == first


def test_kexp_restatement_is_bit_exact():
    xs = np.concatenate([np.linspace(-90, 0, 4001, dtype=np.float32), np.float32([-0.0, -1e-30, -87.0, -86.99])])
    # ko_exp_f32 is reached through a one-cell vote: the weight of a single voter against an absent-free row of two
    for x in xs:
        _, _, w = OC.weighted_vote(np.int32([[[0, 1]]]), np.float32([[0.0, x]]))
        e = W.kexp_np(np.float32(x))
        assert np.float32(w[0]).view(np.uint32) == np.float32(np.float32(1.0) / np.float32(np.float32(1.0) + e)).view(np.uint32)


def test_known_answers():
    ln3 = float(np.log(3.0))
    # n = 3: A against B, B.  A's sum higher by ln 3: each B weighs 1/3, A wins with 1 / (1 + 2/3) = 0.6
    v, c = W.consensus(["A", "B", "B"], np.float32([0.0, -ln3, -ln3]))
    assert (v, c) == ("A", 0.6)
    # higher by less than ln 2: the two Bs outweigh A
    v, c = W.consensus(["A", "B", "B"], np.float32([0.0, -0.5, -0.5]))
    assert v == "B"
    # equal sums: the count vote's winner, ties to the first seen; the likelihood divides by the VOTING weight
    assert W.consensus(["x", "y", "y"], np.float32([-2.0, -2.0, -2.0])) == ("y", round(2 / 3, 5))
    assert W.consensus(["x", "y", None, None], np.float32([-1.0] * 4))[0] == "x"
    assert W.consensus(["x", "y", None, None], np.float32([-1.0] * 4))[1] == 0.5  # count vote: 1 / 4 = 0.25
    # first-seen original of the winning class
    assert W.consensus(["Paris", "paris ", "Rome"], np.float32([-5.0, -0.1, -0.2]))[0] == "Paris"
    # bools: None votes False
    assert W.consensus([True, None, None], np.float32([0.0, -3.0, -3.0]))[0] is True
    assert W.consensus([True, None, None], np.float32([-3.0, 0.0, 0.0]))[0] is False


def test_equal_sums_give_the_count_winner():
    rng = np.random.default_rng(7)
    for _ in range(200):
        n = int(rng.integers(2, 9))
        vals = [str(x) if x >= 0 else None for x in rng.integers(-1, 3, n)]
        if all(v is None for v in vals):
            continue
        seq = np.full(n, np.float32(rng.uniform(-50, 0)), dtype=np.float32)
        assert W.consensus(vals, seq)[0] == O.vote(vals)[0]


# ----------------------------------------------------------------------------- the planner, with the oracle in K3b's place

def _oracle_run(plan, device=None):
    out = {}
    if plan.vote_rows:
        assert plan.weighted
        codes = np.asarray(plan.vote_rows, dtype=np.int32)
        seq = np.asarray(plan.seq_logprobs, dtype=np.float32).reshape(-1, plan.n)
        _, meta, weight = OC.weighted_vote(codes[:, None, :], seq[np.asarray(plan.vote_record)])
        out["vote_meta"], out["vote_weight"] = meta, weight
    if plan.num_rows:
        out["num_value"], out["num_meta"] = OC.numeric(np.asarray(plan.num_rows, dtype=np.float64), plan.rel_eps, plan.abs_eps)
    if plan.medoid_groups:
        out["medoid_idx"], out["medoid_avg"] = OC.medoid(plan.medoid_groups)
    return out


def _oracle_native_consolidate(records, rel_eps, abs_eps, device=0, seq_logprobs=None, counts=None, flags=0):
    """consolidation._native_consolidate with the device JSON path's phases on the host and the oracle in the kernels' place."""
    pairs, _ = jsongpu_with_oracle(records, seq_logprobs, flags=flags)
    if counts is not None:
        counts["device"] = counts.get("device", 0) + sum(p is not None for p in pairs)
    return pairs


@pytest.fixture
def oracle_kernels(monkeypatch):
    from k_llms_b200 import columnar
    from k_llms_b200.utils import consolidation
    monkeypatch.setattr(columnar.Plan, "run", _oracle_run)
    monkeypatch.setattr(consolidation, "_logprob_sums", lambda flat, off: OC.logprob_sum(flat, off))
    monkeypatch.setattr(consolidation, "_native_consolidate", _oracle_native_consolidate)


_WORDS = ["paid", "Paid ", "open", "OPEN", "late", "x", "net 30", "due now"]
_PHRASES = ["payment within thirty days", "payment within 30 days", "pay in thirty days", "net thirty days please"]


def _scalar(rng, kind):
    r = rng.random()
    if r < 0.12:
        return None
    if kind == "enum":
        return _WORDS[int(rng.integers(0, len(_WORDS)))]
    if kind == "bool":
        return bool(rng.integers(0, 2)) if r > 0.25 else None
    if kind == "num":
        return float(rng.choice([10.0, 10.1, 11.0, 250.0]))
    return _PHRASES[int(rng.integers(0, len(_PHRASES)))]


def random_record(rng, n):
    """n candidates of a nested schema: enums, bools with None, numbers, phrases, a sub-object some candidates lack or
    replace by a string, and a list of objects / scalars."""
    out = []
    for _ in range(n):
        d = {"status": _scalar(rng, "enum"), "flag": _scalar(rng, "bool"), "total": _scalar(rng, "num"),
             "note": _scalar(rng, "phrase")}
        r = rng.random()
        if r < 0.6:
            d["addr"] = {"city": _scalar(rng, "enum"), "ok": _scalar(rng, "bool")}
        elif r < 0.8:
            d["addr"] = "unknown"  # not a dict at this node: an absent cell below it
        if rng.random() < 0.7:
            d["items"] = [{"sku": _scalar(rng, "enum"), "paid": _scalar(rng, "bool")} for _ in range(int(rng.integers(0, 3)))]
        if rng.random() < 0.3:
            d["tags"] = [_scalar(rng, "enum") for _ in range(int(rng.integers(1, 3)))]
        if rng.random() < 0.1:
            d = "not an object"
        out.append(d)
    return out


def _seq(rng, n):
    k = rng.random()
    if k < 0.2:
        return np.full(n, np.float32(-3.25))
    if k < 0.3:
        return rng.choice([-9999.0, -1.0], n).astype(np.float32)
    return (-rng.exponential(4.0, n)).astype(np.float32)


@pytest.mark.parametrize("allow_none", [False, True])
def test_planner_matches_weighted_oracle(oracle_kernels, allow_none):
    from k_llms_b200.utils.consensus_utils import ConsensusSettings, consensus_values, consensus_values_batch
    rng = np.random.default_rng(11 + allow_none)
    settings = ConsensusSettings(allow_none_as_candidate=allow_none)
    osettings = O.OracleSettings(allow_none_as_candidate=allow_none)
    records, seqs = [], []
    for _ in range(150):
        n = int(rng.choice([1, 2, 3, 5, 8, 16]))
        records.append(random_record(rng, n))
        seqs.append(_seq(rng, n))
    expected = [W.consensus(v, s, osettings, 1.0, EMBED) for v, s in zip(records, seqs)]
    for v, s, e in zip(records, seqs, expected):
        got = consensus_values(v, settings, EMBED, None, seq_logprobs=s)
        assert same(got, e), (v, s, got, e)
    # one plan for the whole batch: rows padded to the widest record
    n_max = max(len(r) for r in records)
    padded = np.full((len(records), n_max), np.float32(7.0), dtype=np.float32)  # entries past a record's candidates are ignored
    for r, s in enumerate(seqs):
        padded[r, :len(s)] = s
    got = consensus_values_batch(records, settings, EMBED, None, seq_logprobs=padded)
    for g, e in zip(got, expected):
        assert same(g, e)


def test_cells_stay_at_candidate_positions(oracle_kernels):
    """Below a node where candidate 1 is not a dict, cell i is candidate i.  Compacting the dicts would put candidates 2 and
    3 into cells 1 and 2 and give them the weights of candidates 1 and 2."""
    from k_llms_b200.utils.consensus_utils import ConsensusSettings, consensus_values
    values = [{"k": "b"}, "zzz", {"k": "c"}, {"k": "c"}]
    for seq, winner in ((np.float32([0.0, -9999.0, -0.5, -0.5]), "c"),   # compacted: b 1 against c ~0 + e^-0.5
                        (np.float32([0.0, 0.0, -1.0, -1.0]), "b")):       # compacted: b 1 against c 1 + e^-1
        got = consensus_values(values, ConsensusSettings(), EMBED, None, seq_logprobs=seq)
        assert got[0] == {"k": winner}
        assert same(got, W.consensus(values, seq, O.DEFAULTS, 1.0, EMBED))
        # the same one level down, and in a list
        got = consensus_values([{"a": v} for v in values], ConsensusSettings(), EMBED, None, seq_logprobs=seq)
        assert got[0] == {"a": {"k": winner}}
        got = consensus_values([[v] if isinstance(v, dict) else v for v in values], ConsensusSettings(), EMBED, None, seq_logprobs=seq)
        assert got[0] == [{"k": winner}]


# ----------------------------------------------------------------------------- consolidation entry points and input checks

def _completion(contents, logprobs):
    from openai.types.chat import ChatCompletion
    choices = []
    for i, (c, lp) in enumerate(zip(contents, logprobs)):
        ch = {"index": i, "finish_reason": "stop", "message": {"role": "assistant", "content": c}, "logprobs": None}
        if lp is not None:
            ch["logprobs"] = {"content": [{"token": "t", "logprob": x, "bytes": None, "top_logprobs": []} for x in lp]}
        choices.append(ch)
    return ChatCompletion.model_validate({"id": "x", "object": "chat.completion", "created": 0, "model": "m", "choices": choices})


def test_consolidate_chat_completions_weighted(oracle_kernels):
    import json
    from k_llms_b200.utils.consolidation import consolidate_chat_completions
    texts = [json.dumps({"s": "A", "n": 1}), "", json.dumps({"s": "B", "n": 1}), json.dumps({"s": "B", "n": 2})]
    lps = [[-0.1, -0.2], None, [-3.0, -1.0], [-2.5, -2.0]]  # the empty choice is not a candidate: its logprobs are not needed
    out = consolidate_chat_completions(_completion(texts, lps), EMBED, None, vote_weighting="likelihood")
    seq = OC.logprob_sum(np.float32([-0.1, -0.2, -3.0, -1.0, -2.5, -2.0]), np.int64([0, 2, 4, 6]))
    exp = W.client_order([json.loads(t) for t in texts if t], seq, O.DEFAULTS, EMBED)
    assert json.loads(out.choices[0].message.content) == exp[0] and out.likelihoods == exp[1]
    assert exp[0]["s"] == "A"


@pytest.mark.parametrize("bad", [None, "no_content", [math.nan], [-math.inf], [math.inf], [-1e39]])
def test_input_checks(oracle_kernels, bad, monkeypatch):
    import json
    from k_llms_b200.utils import consolidation
    from k_llms_b200.utils.consolidation import consolidate_chat_completions, consolidate_contents_batch

    def no_gpu(*a, **k):
        raise AssertionError("GPU work before the input check")
    monkeypatch.setattr(consolidation, "_logprob_sums", no_gpu)
    texts = [json.dumps({"s": "A"}), json.dumps({"s": "B"})]
    comp = _completion(texts, [[-0.1], [-0.2]])
    if bad == "no_content":
        comp.choices[1].logprobs.content = None
    else:
        comp.choices[1].logprobs = None if bad is None else comp.choices[1].logprobs.model_copy(update={
            "content": [comp.choices[1].logprobs.content[0].model_copy(update={"logprob": bad[0]})]})
    with pytest.raises(ValueError):
        consolidate_chat_completions(comp, EMBED, None, vote_weighting="likelihood")
    if bad != "no_content":
        with pytest.raises(ValueError):
            consolidate_contents_batch([texts], token_logprobs=[[[-0.1], bad]])


def test_contents_batch_weighted(oracle_kernels):
    import json
    from k_llms_b200.utils.consolidation import consolidate_contents_batch
    rng = np.random.default_rng(5)
    records, lps, exp = [], [], []
    for _ in range(60):
        n = int(rng.choice([1, 2, 3, 5]))
        cands = random_record(rng, n)
        texts = [json.dumps(c) if rng.random() > 0.1 else "" for c in cands]
        toks = [list((-rng.exponential(1.0, int(rng.integers(0, 6)))).astype(np.float64)) for _ in texts]
        records.append(texts)
        lps.append(toks)
    got = consolidate_contents_batch(records, token_logprobs=lps)
    from k_llms_b200.utils.consolidation import _aligned_sync, _format_consensus_content, _safe_parse_content
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    for texts, toks, g in zip(records, lps, got):
        if len(texts) == 1:
            assert g == (texts[0], None)
            continue
        keep = [c for c, t in enumerate(texts) if t]
        flat = np.float32([x for c in keep for x in toks[c]])
        off = np.int64([0] + list(np.cumsum([len(toks[c]) for c in keep])))
        seq = OC.logprob_sum(flat, off)
        contents = [_safe_parse_content(texts[c]) for c in keep]
        aligned = _aligned_sync(contents, ConsensusSettings(), EMBED, None)
        value, conf = W.client_order(contents, seq, O.DEFAULTS, EMBED, aligned=aligned)
        assert g[0] == _format_consensus_content(value) and same(g[1], conf), (texts, g, value, conf)


# ----------------------------------------------------------------------------- the client keyword

class _Recorder:
    """A stand-in OpenAI client: records the parameters and answers with a fixed completion."""

    def __init__(self, completion, is_async=False):
        self.calls, self._c, self._async = [], completion, is_async
        self.chat = type("C", (), {"completions": self})()
        self.beta = type("B", (), {"chat": self.chat})()

    def create(self, **params):
        self.calls.append(params)
        if self._async:
            async def ret():
                return self._c
            return ret()
        return self._c

    def parse(self, **params):
        from openai.types.chat import ParsedChatCompletion
        self.calls.append(params)
        pc = ParsedChatCompletion.model_validate(self._c.model_dump())
        if self._async:
            async def ret():
                return pc
            return ret()
        return pc


def _wrapped(is_async, completion):
    from k_llms_b200.client import AsyncKLLMs, KLLMs
    w = (AsyncKLLMs if is_async else KLLMs)(api_key="k")
    rec = _Recorder(completion, is_async)
    w._client = rec
    if is_async:
        async def emb(texts, model, batch, verbose):
            return [[0.0] for _ in texts]
        w.get_embeddings = emb
    else:
        w.get_embeddings = lambda texts, model, batch, verbose: [[0.0] for _ in texts]
    return w, rec


@pytest.mark.parametrize("is_async", [False, True])
@pytest.mark.parametrize("method", ["create", "parse"])
def test_client_keyword(oracle_kernels, is_async, method):
    import json
    comp = _completion([json.dumps({"s": "A"}), json.dumps({"s": "B"}), json.dumps({"s": "B"})], [[0.0], [-2.0], [-2.0]])
    w, rec = _wrapped(is_async, comp)
    call = getattr(w.chat.completions, method)
    kw = dict(messages=[{"role": "user", "content": "q"}], model="m", n=3)
    if method == "parse":
        kw["response_format"] = None
    run = (lambda r: asyncio.run(r)) if is_async else (lambda r: r)
    out = run(call(**kw, vote_weighting="likelihood"))
    assert rec.calls[-1]["logprobs"] is True and "vote_weighting" not in rec.calls[-1]
    assert json.loads(out.choices[0].message.content) == {"s": "A"}  # 1 against 2 x e^-2
    with pytest.raises(ValueError):
        run(call(**kw, vote_weighting="likelihood", logprobs=False))
    assert len(rec.calls) == 1  # refused before the API call
    with pytest.raises(ValueError):
        run(call(**kw, vote_weighting="votes"))
    assert len(rec.calls) == 1


def test_client_default_request_unchanged():
    from k_llms_b200.resources.completions.completions import _call_params
    base = {"messages": [], "model": "m"}
    assert _call_params(base, {"temperature": 0.5}, 4, {}) == _call_params(base, {"temperature": 0.5}, 4, {}, "count")
    assert "logprobs" not in _call_params(base, {}, 4, {})
    assert _call_params(base, {}, 4, {"logprobs": True, "top_logprobs": 2}, "count")["logprobs"] is True
    assert _call_params(base, {}, 4, {}, "likelihood")["logprobs"] is True


# ----------------------------------------------------------------------------- the weighted device JSON path's phases on the host

def _flat_records(rng, R, n):
    """Records the device path models (flat objects of one key sequence) and ones it declines (nested values, lists, other keys,
    multi-word strings, escapes)."""
    out = []
    for r in range(R):
        cands = []
        shape = rng.random()
        for _ in range(n):
            d = {"status": _WORDS[int(rng.integers(0, 4))] if rng.random() > 0.1 else None,
                 "flag": bool(rng.integers(0, 2)) if rng.random() > 0.15 else None,
                 "code": str(rng.choice(["A1", "a1", "B2", "b 2"])),
                 "total": float(rng.choice([10.0, 10.1, 11.0])) if rng.random() > 0.1 else None}
            if shape < 0.1:
                d["addr"] = {"city": "x"}
            elif shape < 0.2:
                d["items"] = [1, 2]
            elif shape < 0.25:
                d["note"] = str(rng.choice(["pay within thirty days", "pay in 30 days"]))
            elif shape < 0.3 and rng.random() < 0.5:
                d = {"other": 1}
            cands.append(json.dumps(d))
        out.append(cands)
    return out


@pytest.mark.parametrize("n", [2, 3, 5, 8, 16])
def test_weighted_device_phases_match_planner(oracle_kernels, n):
    """kc_consolidate_json_packed_weighted's phases on the host (oracle in K3b's place) against the weighted Python planner,
    byte for byte; the records it declines are exactly the ones the count-vote device path declines."""
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from k_llms_b200.utils.consolidation import _aligned_sync, _format_consensus_content, _safe_parse_content
    rng = np.random.default_rng(400 + n)
    records = _flat_records(rng, 300, n)
    seq = np.concatenate([_seq(rng, n) for _ in records]).astype(np.float32)
    pairs, status = jsongpu_with_oracle(records, seq)
    _, status_count = jsongpu_with_oracle(records)
    assert [s != 0 for s in status] == [s != 0 for s in status_count]
    assert sum(p is not None for p in pairs) > 150
    for r, (texts, p) in enumerate(zip(records, pairs)):
        if p is None:
            continue
        contents = [_safe_parse_content(t) for t in texts]
        aligned = _aligned_sync(contents, ConsensusSettings(), EMBED, None)
        value, conf = W.client_order(contents, seq[r * n:(r + 1) * n], O.DEFAULTS, EMBED, aligned=aligned)
        assert p == (_format_consensus_content(value), json.dumps(conf)), (texts, p, value, conf)


def test_contents_batch_counts_device_records(oracle_kernels):
    from k_llms_b200.utils.consolidation import consolidate_contents_batch
    rng = np.random.default_rng(9)
    records = _flat_records(rng, 40, 3) + [["", json.dumps({"a": "x"}), json.dumps({"a": "y"})]]
    lps = [[list(-rng.exponential(1.0, 3)) for _ in t] for t in records]
    counts = {}
    got = consolidate_contents_batch(records, token_logprobs=lps, counts=counts)
    assert 20 <= counts["device"] <= len(records) and len(got) == len(records)
