"""Consolidation glue: n choices -> align -> consensus -> choices[0] = consensus, choices[1..n] = originals.

Same four entry points, signatures and result shape as reference k_llms/utils/consolidation.py:63-493; the four
near-identical bodies there share one implementation here.  The consensus itself runs on the GPU
(`consensus_utils.consensus_values`); JSON parsing and object rebuilding stay host Python (SURVEY.md §8a a8).
"""
from __future__ import annotations

import asyncio
import json
from typing import Any, List, Literal, Optional, Sequence, Union

from openai.types.chat import ChatCompletion, ChatCompletionMessage, ParsedChatCompletion
from openai.types.chat.chat_completion import Choice
from openai.types.chat.parsed_chat_completion import ParsedChatCompletionMessage, ParsedChoice
from pydantic import BaseModel

from ..types.completions import KLLMsChatCompletion
from ..types.parsed import KLLMsParsedChatCompletion
from .consensus_utils import (
    ASYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    ConsensusSettings,
    async_consensus_values,
    async_recursive_list_alignments,
    consensus_values,
    recursive_list_alignments,
)


def _safe_parse_content(content: str) -> dict:
    """JSON if it parses, else {"text": content} (reference consolidation.py:25-38)."""
    try:
        return json.loads(content)
    except (json.JSONDecodeError, TypeError):
        return {"text": content}


def _format_consensus_content(consensus_content: Any) -> str:
    """Inverse of _safe_parse_content for the consensus message (reference consolidation.py:41-60)."""
    if consensus_content is None:
        return ""
    if isinstance(consensus_content, dict) and len(consensus_content) == 1 and isinstance(consensus_content.get("text"), str):
        return consensus_content["text"]
    return json.dumps(consensus_content)


def _contents_of(choices) -> List[dict]:
    return [_safe_parse_content(c.message.content) for c in choices if c.message.content]


# ----------------------------------------------------------------------------- likelihood weighting (DESIGN.md §5)

VOTE_WEIGHTINGS = ("count", "likelihood")


def _check_weighting(vote_weighting: str) -> bool:
    """True for likelihood weighting."""
    if vote_weighting not in VOTE_WEIGHTINGS:
        raise ValueError(f"vote_weighting={vote_weighting!r}: expected one of {VOTE_WEIGHTINGS}")
    return vote_weighting == "likelihood"


def _token_logprobs_of(choices) -> List[List[float]]:
    """The token logprobs of the candidates — the choices `_contents_of` keeps, in the same order."""
    out = []
    for i, c in enumerate(choices):
        if not c.message.content:
            continue
        lp = getattr(c, "logprobs", None)
        if lp is None or lp.content is None:
            raise ValueError(f"vote_weighting='likelihood' needs the token logprobs of every candidate; choice {i} has none "
                             "(request them with logprobs=True)")
        out.append([t.logprob for t in lp.content])
    return out


def _pack_logprobs(seqs: List[List[float]]):
    """Every candidate's token logprobs as K3's input (float32 [T], int64 offsets [S+1]).  Missing or non-finite (as float32)
    logprobs raise ValueError — before anything runs on the GPU."""
    import numpy as np
    for s, seq in enumerate(seqs):
        if seq is None:
            raise ValueError(f"vote_weighting='likelihood' needs the token logprobs of every candidate; candidate {s} has none")
    lens = np.fromiter((len(seq) for seq in seqs), dtype=np.int64, count=len(seqs))
    offsets = np.zeros(len(seqs) + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    with np.errstate(over="ignore"):  # a logprob beyond the float32 range becomes inf and is refused below
        flat = np.fromiter((float(x) for seq in seqs for x in seq), dtype=np.float64, count=int(offsets[-1])).astype(np.float32)
    if not np.isfinite(flat).all():
        bad = int(np.searchsorted(offsets, int(np.flatnonzero(~np.isfinite(flat))[0]), side="right")) - 1
        raise ValueError(f"token logprobs must be finite (as float32); candidate {bad} has {seqs[bad]!r}")
    return flat, offsets


def _sequence_logprobs(seqs: List[List[float]]) -> List[float]:
    """K3 (kc_logprob_sum_f32) over every candidate's token logprobs in ONE launch: their fp32 sums, in order (checked first,
    _pack_logprobs)."""
    flat, offsets = _pack_logprobs(seqs)
    if not seqs:
        return []
    return [float(x) for x in _logprob_sums(flat, offsets)]


def _logprob_sums(flat, offsets):
    """K3 on the current device: float32 token logprobs [T], int64 offsets [S+1] -> float32 sums [S] (numpy)."""
    from .. import _native
    torch = _native._require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    return _native.logprob_sum(torch.from_numpy(flat).to(dev), torch.from_numpy(offsets).to(dev)).cpu().numpy()


def _native_alignment(contents, settings):
    """The alignment pre-pass in native code (H2, `kc_align_json`: same result as `recursive_list_alignments`, pinned on the
    reference's goldens) — or None when the record needs the Python pre-pass: another similarity method than the default,
    string pairs that go to the embeddings service (both longer than 50 characters), non-ASCII text."""
    if settings.string_similarity_method != "embeddings":
        return None
    from .. import _native
    return _native.align_json(contents, settings.min_support_ratio)


def _native_settings(settings) -> bool:
    """The settings the native JSON path (H1, kc_consolidate_json) implements: the reference's defaults."""
    return (not settings.allow_none_as_candidate and settings.string_similarity_method == "embeddings"
            and settings.string_consensus_method == "centroid" and settings.min_support_ratio == 0.51)


def _native_request(choices, settings, embed, weighted: bool):
    """(candidate texts, their token logprobs or None) of a request the native JSON path may take, or None when it needs the
    Python path (non-default settings, fewer than two or more than 64 non-empty contents; no embeddings callable: the reference
    raises ValueError for primitive fields then, cu:1445-1446, and so does the Python path)."""
    from .. import _native
    # weighted: the token logprobs of the same candidates, checked before anything runs on the GPU
    lp = _pack_logprobs(_token_logprobs_of(choices)) if weighted else None
    if embed is None:
        return None
    texts = [c.message.content for c in choices if c.message.content]  # the filter of _contents_of (reference consolidation.py:92)
    if len(texts) < 2 or len(texts) > _native.MAX_CANDIDATES or not _native_settings(settings):
        return None
    return texts, lp


def _consensus_of_choices_native(choices, settings, embed, weighted: bool = False):
    """The whole per-request path in native code (H1): the n `choice.message.content` texts in -> (consensus value,
    likelihoods), i.e. parse + alignment pre-pass + vote / numeric / medoid kernels + decode — or None when the request needs
    the Python path (_native_request's rules, anything H1 declines)."""
    req = _native_request(choices, settings, embed, weighted)
    if req is None:
        return None
    return _native_value(_combiner.run(req[0], settings.rel_eps, settings.abs_eps, req[1]))


async def _consensus_of_choices_native_async(choices, settings, embed, weighted: bool = False):
    """The async twin of _consensus_of_choices_native: the device JSON path with the reference's ASYNC dispatcher
    (JSON_NUMERIC_MEDOID: numeric fields are similarity medoids, K5).  None when the request needs the Python async route:
    _native_request's rules, no CUDA device, or anything the device path declines (it hands nothing to the host path H1, which
    decides numbers the sync way).  The event loop is not blocked while the GPU works."""
    import torch
    from .. import _native
    if not torch.cuda.is_available():
        return None
    req = _native_request(choices, settings, embed, weighted)
    if req is None:
        return None
    return _native_value(await _combiner.run_async(req[0], settings.rel_eps, settings.abs_eps, req[1], _native.JSON_NUMERIC_MEDOID))


def _native_value(out):
    """(consensus value, likelihoods) of one record's native result texts, or None."""
    if out is None:
        return None
    content_text, likelihoods_text = out
    try:  # undo _format_consensus_content: a consensus that is not a JSON object is the unwrapped {"text": s}
        value = json.loads(content_text)
    except ValueError:
        value = None
    if not isinstance(value, dict):
        value = {"text": content_text}
    return value, json.loads(likelihoods_text)


def _native_consolidate(records, rel_eps, abs_eps, device: int = 0, seq_logprobs=None, counts=None, flags: int = 0):
    """records of n candidate texts -> [(content, likelihoods text) or None]: the device JSON path (H1g,
    kc_consolidate_json_packed: scan / key sort / typing / encode / K1 + K2 / emit on the GPU; re-entrant, pooled streams), which
    hands what it does not model to the host path (H1, kc_consolidate_json) inside the same call.  seq_logprobs (float32
    [R*n], the candidates' sums): likelihood-weighted votes (kc_consolidate_json_packed_weighted; no host path).  flags:
    _native.JSON_NUMERIC_MEDOID for the async dispatcher (no host path either).  Records whose candidates differ in shape (key
    order, missing or extra keys, null sub-objects) stay on the device (JSON_KEY_UNION, always set here), and so do records with
    list fields (JSON_LISTS: the alignment pre-pass on host threads, then the aligned texts on the device), and so do records
    whose similarity-medoid fields hold non-ASCII text or \\uXXXX escapes (JSON_UNICODE).  counts (optional dict): "device" +=
    the records the device path consolidated."""
    from .. import _native
    blob, off, n = _native.pack_texts(records, pinned=len(records) >= 256)  # page-locking only pays for batches
    flags |= _native.JSON_KEY_UNION | _native.JSON_LISTS | _native.JSON_UNICODE
    if seq_logprobs is None:
        res = _native.consolidate_json_packed(blob, off, n, rel_eps, abs_eps, device, flags=flags)
    else:
        res = _native.consolidate_json_packed_weighted(blob, off, n, seq_logprobs, rel_eps, abs_eps, device, flags=flags)
    try:
        if counts is not None:
            counts["device"] = counts.get("device", 0) + int(res.stats.n_device)
        return res.pairs()
    finally:
        res.close()


class _Combiner:
    """Per-request consolidations that arrive while another one is on the GPU are COMBINED into one batched call (flat
    combining: the thread that holds the device runs its own request, then everything that queued up meanwhile as one
    kc_consolidate_json_packed call, and hands the results back).  An idle caller pays nothing (it takes the device and runs
    directly); under load the cost per request falls from one launch sequence each towards the batched rate
    (tools/latency.py: tens of thousands of requests per second).  Coroutines queue through run_async, which never blocks the
    event loop: the device is driven from a helper thread that completes the coroutines' futures.  Requests are combined per
    (candidate count, eps, weighted, flags)."""

    def __init__(self):
        import threading
        self._device = threading.Lock()
        self._qlock = threading.Lock()
        self._queue: list = []
        self._helper = None  # the one thread that drives the device for coroutines (created on first use)

    def _drain(self):
        while True:
            with self._qlock:
                batch, self._queue = self._queue, []
            if not batch:
                return
            groups: dict = {}
            for item in batch:  # weighted requests apart from count votes, async dispatcher (flags) apart from sync
                groups.setdefault((len(item["texts"]), item["eps"], item["lp"] is not None, item["flags"]), []).append(item)
            for (_n, eps, weighted, flags), items in groups.items():
                try:
                    seq = None
                    if weighted:  # one K3 launch for the whole combined call
                        import numpy as np
                        flat = np.concatenate([it["lp"][0] for it in items])
                        offs, base = [np.zeros(1, dtype=np.int64)], 0
                        for it in items:
                            offs.append(it["lp"][1][1:] + base)
                            base += int(it["lp"][1][-1])
                        seq = _logprob_sums(flat, np.concatenate(offs))
                    extra = {"flags": flags} if flags else {}  # the sync calls keep their signature
                    outs = _native_consolidate([it["texts"] for it in items], eps[0], eps[1], seq_logprobs=seq, **extra)
                    for it, o in zip(items, outs):
                        it["out"] = o
                except BaseException as exc:  # hand the failure to every waiter of the group
                    for it in items:
                        it["err"] = exc
                for it in items:
                    it["notify"]()

    def _serve(self, held: bool = False):
        """Drain while the device is free (held: the caller has already taken it).  After releasing it, look again: an item
        queued while this thread held the device, whose caller found the device taken, is then served here or by the thread
        that took the device since."""
        while held or self._device.acquire(blocking=False):
            held = False
            try:
                self._drain()
            finally:
                self._device.release()
            with self._qlock:
                if not self._queue:
                    return

    def _enqueue(self, texts, rel_eps, abs_eps, lp, flags, notify):
        item = {"texts": texts, "eps": (rel_eps, abs_eps), "lp": lp, "flags": flags, "notify": notify, "out": None, "err": None}
        with self._qlock:
            self._queue.append(item)
        return item

    @staticmethod
    def _result(item):
        if item["err"] is not None:
            raise item["err"]
        return item["out"]

    def run(self, texts, rel_eps, abs_eps, lp=None, flags: int = 0):
        """lp: (token logprobs, offsets) of the texts (_pack_logprobs) for likelihood-weighted votes, or None; flags: those of
        kc_consolidate_json_packed."""
        import threading
        done = threading.Event()
        item = self._enqueue(texts, rel_eps, abs_eps, lp, flags, done.set)
        while not done.is_set():
            self._serve()
            if not done.is_set():
                done.wait(0.0005)
        return self._result(item)

    async def run_async(self, texts, rel_eps, abs_eps, lp=None, flags: int = 0):
        """run() for a coroutine.  If the device is free, the helper thread drains the queue (this request and whatever queues up
        meanwhile); else the thread holding the device serves it.  The coroutine waits on a future of its loop."""
        loop = asyncio.get_running_loop()
        fut = loop.create_future()

        def wake():
            if not fut.done():
                fut.set_result(None)

        def notify():
            try:
                loop.call_soon_threadsafe(wake)
            except RuntimeError:  # the loop has been closed: nobody waits for the result
                pass

        item = self._enqueue(texts, rel_eps, abs_eps, lp, flags, notify)
        if self._device.acquire(blocking=False):
            if self._helper is None:  # one worker is enough: only the thread that took the device hands it work
                from concurrent.futures import ThreadPoolExecutor
                self._helper = ThreadPoolExecutor(max_workers=1, thread_name_prefix="kllms-combiner")
            self._helper.submit(self._serve, True)
        await fut
        return self._result(item)


_combiner = _Combiner()


def _check_candidates(n: int) -> None:
    from .. import _native
    if n > _native.MAX_CANDIDATES:
        raise ValueError(f"{n} candidates in one request: k_llms_b200 consolidates at most {_native.MAX_CANDIDATES} "
                         "(README.md, Limits)")


def _aligned_sync(contents, settings, embed, client):
    if len(contents) >= 2:  # reference consolidation.py:96-104
        aligned = _native_alignment(contents, settings)
        if aligned is None:
            aligned, _ = recursive_list_alignments(contents, settings.string_similarity_method, embed, client, settings.min_support_ratio)
        contents = [(d if isinstance(d, dict) else {}) for d in aligned]
    return contents


def _consensus_sync(contents, settings, embed, client, seq_logprobs=None):
    """seq_logprobs: the candidates' sequence logprobs for a likelihood-weighted vote, or None (the alignment keeps every
    candidate at its position, so sum c stays with candidate c)."""
    return consensus_values(_aligned_sync(contents, settings, embed, client), settings, embed, client=client, seq_logprobs=seq_logprobs)


async def _consensus_async(contents, settings, embed, client, seq_logprobs=None):
    if len(contents) >= 2:
        aligned = _native_alignment(contents, settings)
        if aligned is None:
            aligned, _ = await async_recursive_list_alignments(contents, settings.string_similarity_method, embed, client,
                                                               settings.min_support_ratio)
        contents = [(d if isinstance(d, dict) else {}) for d in aligned]
    return await async_consensus_values(contents, settings, embed, client=client, seq_logprobs=seq_logprobs)


def _weighted_contents(choices):
    """(contents, their sequence logprobs) of a likelihood-weighted request: the logprobs are checked before any GPU work."""
    return _contents_of(choices), _sequence_logprobs(_token_logprobs_of(choices))


def _consensus_of_choices_python(choices, settings, embed, client, weighted: bool):
    """The Python planner's consensus of the choices (what the native path leaves to it), weighted or not."""
    contents, sums = _weighted_contents(choices) if weighted else (_contents_of(choices), None)
    return _consensus_sync(contents, settings, embed, client, sums)


async def _consensus_of_choices_async(choices, settings, embed, client, weighted: bool):
    """The async entry points' consensus of the choices: the device JSON path with the async dispatcher's numeric medoid when it
    takes the request, else the Python async route (async_consensus_values: the reference's async semantics, votes on the GPU)."""
    native = await _consensus_of_choices_native_async(choices, settings, embed, weighted)
    if native is not None:
        return native
    contents, sums = _weighted_contents(choices) if weighted else (_contents_of(choices), None)
    return await _consensus_async(contents, settings, embed, client, sums)


def _assemble_plain(base: ChatCompletion, heads, consensus_content, likelihoods) -> KLLMsChatCompletion:
    """heads: the choices whose message/finish_reason/logprobs become choices[1..]; heads[0] lends its
    function_call / tool_calls / refusal / finish_reason / logprobs to the consensus choice."""
    first = heads[0] if heads else None
    message = ChatCompletionMessage(
        role="assistant",
        content=_format_consensus_content(consensus_content),
        function_call=first.message.function_call if first else None,
        tool_calls=first.message.tool_calls if first else None,
        refusal=first.message.refusal if first else None,
    )
    consensus_choice = Choice(finish_reason=first.finish_reason if first else "stop", index=0, message=message,
                              logprobs=first.logprobs if first else None)
    originals = [Choice(finish_reason=c.finish_reason, index=i + 1, message=c.message, logprobs=c.logprobs)
                 for i, c in enumerate(heads)]
    return KLLMsChatCompletion.model_validate(
        {**base.model_dump(), "choices": [consensus_choice] + originals, "likelihoods": likelihoods, "usage": base.usage})


def consolidate_chat_completions(
    completions: Union[List[ChatCompletion], ChatCompletion],
    get_openai_embeddings_from_text: SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    consensus_settings: ConsensusSettings = ConsensusSettings(),
    vote_weighting: Literal["count", "likelihood"] = "count",
) -> KLLMsChatCompletion:
    """One ChatCompletion with n choices, or a list of completions (reference consolidation.py:63-216).
    vote_weighting="likelihood": the str / bool vote leaves weigh each candidate by the likelihood of its choice, from
    `choice.logprobs.content[i].logprob` (DESIGN.md §5, self-defined); everything else is decided as with "count"."""
    weighted = _check_weighting(vote_weighting)
    if isinstance(completions, ChatCompletion):
        completion = completions
        assert len(completion.choices) > 0, "Cannot consolidate empty list of choices"
        if len(completion.choices) == 1:
            return KLLMsChatCompletion.model_validate(completion.model_dump())
        _check_candidates(len(completion.choices))
        content, likelihoods = (_consensus_of_choices_native(completion.choices, consensus_settings, get_openai_embeddings_from_text, weighted)
                                or _consensus_of_choices_python(completion.choices, consensus_settings, get_openai_embeddings_from_text, client,
                                                                weighted))
        return _assemble_plain(completion, list(completion.choices), content, likelihoods)
    completion_list = completions
    assert len(completion_list) > 0, "Cannot consolidate empty list of completions"
    if len(completion_list) == 1:
        return KLLMsChatCompletion.model_validate(completion_list[0].model_dump())
    _check_candidates(len(completion_list))
    # choices[i + 1] keeps the index of completion i and completion_list[0] lends its head fields (reference consolidation.py:
    # 176-216); a completion without choices contributes nothing
    firsts = [(i, c.choices[0]) for i, c in enumerate(completion_list) if c.choices]
    heads = [c for _, c in firsts]
    content, likelihoods = (_consensus_of_choices_native(heads, consensus_settings, get_openai_embeddings_from_text, weighted)
                            or _consensus_of_choices_python(heads, consensus_settings, get_openai_embeddings_from_text, client, weighted))
    out = _assemble_plain(completion_list[0], heads, content, likelihoods)
    for k, (i, _) in enumerate(firsts):
        out.choices[k + 1].index = i + 1
    return out


async def async_consolidate_chat_completions(
    completion: ChatCompletion,
    async_get_openai_embeddings_from_text: ASYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    consensus_settings: ConsensusSettings = ConsensusSettings(),
    vote_weighting: Literal["count", "likelihood"] = "count",
) -> KLLMsChatCompletion:
    """Reference consolidation.py:219-303; vote_weighting as for consolidate_chat_completions."""
    weighted = _check_weighting(vote_weighting)
    assert len(completion.choices) > 0, "Cannot consolidate empty list of choices"
    if len(completion.choices) == 1:
        return KLLMsChatCompletion.model_validate(completion.model_dump())
    _check_candidates(len(completion.choices))
    content, likelihoods = await _consensus_of_choices_async(completion.choices, consensus_settings, async_get_openai_embeddings_from_text,
                                                             client, weighted)
    return _assemble_plain(completion, list(completion.choices), content, likelihoods)


def _assemble_parsed(completion: ParsedChatCompletion, consensus_content, likelihoods, response_format, keep_usage: bool):
    parsed = None
    if response_format and consensus_content is not None:
        try:  # validation failures are swallowed: parsed stays None (reference consolidation.py:358-365)
            if isinstance(response_format, type) and issubclass(response_format, BaseModel):
                parsed = response_format.model_validate(consensus_content)
        except Exception:
            parsed = None
    first = completion.choices[0]
    message = ParsedChatCompletionMessage(
        role="assistant",
        content=_format_consensus_content(consensus_content),
        function_call=first.message.function_call,
        tool_calls=first.message.tool_calls,
        refusal=first.message.refusal,
        parsed=parsed,
    )
    consensus_choice = ParsedChoice(finish_reason=first.finish_reason, index=0, message=message, logprobs=first.logprobs)
    originals = [ParsedChoice(finish_reason=c.finish_reason, index=i + 1, message=c.message, logprobs=c.logprobs)
                 for i, c in enumerate(completion.choices)]
    payload = {**completion.model_dump(), "choices": [consensus_choice] + originals, "likelihoods": likelihoods}
    if keep_usage:
        payload["usage"] = completion.usage
    return KLLMsParsedChatCompletion.model_validate(payload)


def consolidate_parsed_chat_completions(
    completion: ParsedChatCompletion,
    get_openai_embeddings_from_text: SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    consensus_settings: ConsensusSettings = ConsensusSettings(),
    response_format: Optional[type] = None,
    vote_weighting: Literal["count", "likelihood"] = "count",
) -> KLLMsParsedChatCompletion:
    """Reference consolidation.py:306-399; vote_weighting as for consolidate_chat_completions."""
    weighted = _check_weighting(vote_weighting)
    assert len(completion.choices) > 0, "Cannot consolidate empty list of choices"
    if len(completion.choices) == 1:
        return KLLMsParsedChatCompletion.model_validate(completion.model_dump())
    _check_candidates(len(completion.choices))
    content, likelihoods = (_consensus_of_choices_native(completion.choices, consensus_settings, get_openai_embeddings_from_text, weighted)
                            or _consensus_of_choices_python(completion.choices, consensus_settings, get_openai_embeddings_from_text, client,
                                                            weighted))
    return _assemble_parsed(completion, content, likelihoods, response_format, keep_usage=True)


async def async_consolidate_parsed_chat_completions(
    completion: ParsedChatCompletion,
    async_get_openai_embeddings_from_text: ASYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    consensus_settings: ConsensusSettings = ConsensusSettings(),
    response_format: Optional[type] = None,
    vote_weighting: Literal["count", "likelihood"] = "count",
) -> KLLMsParsedChatCompletion:
    """Reference consolidation.py:402-493 (the reference's async twin does not re-attach `usage`; model_dump keeps it);
    vote_weighting as for consolidate_chat_completions."""
    weighted = _check_weighting(vote_weighting)
    assert len(completion.choices) > 0, "Cannot consolidate empty list of choices"
    if len(completion.choices) == 1:
        return KLLMsParsedChatCompletion.model_validate(completion.model_dump())
    _check_candidates(len(completion.choices))
    content, likelihoods = await _consensus_of_choices_async(completion.choices, consensus_settings, async_get_openai_embeddings_from_text,
                                                             client, weighted)
    return _assemble_parsed(completion, content, likelihoods, response_format, keep_usage=False)


def consolidate_contents_batch(records: List[List[str]], consensus_settings: ConsensusSettings = ConsensusSettings(),
                               get_openai_embeddings_from_text: Optional[SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE] = None,
                               client: Any = None, device: int = 0,
                               token_logprobs: Optional[Sequence[Sequence[Optional[Sequence[float]]]]] = None,
                               counts: Optional[dict] = None):
    """Batched consolidation of raw contents (new; the reference has no batch dimension): for every record, the n
    `choice.message.content` strings in -> (consensus content string, likelihoods) out, exactly what the per-request
    functions above put into choices[0] and `likelihoods`.

    token_logprobs[r][c] (optional): the token logprobs of candidate text records[r][c].  Given, the vote leaves are
    likelihood-weighted (DESIGN.md §5), as the per-request functions do with vote_weighting="likelihood": one K3 launch sums
    the candidates' logprobs, the weighted device JSON path (K3b in K1's place) consolidates what it models, and the rest is
    planned in Python with one K3b launch.  counts (optional dict, weighted calls): "device" = the records the device path
    consolidated.

    With the default settings the batch goes to the device JSON path (H1g, kc_consolidate_json_packed: the texts are copied to
    the GPU as they are; scan / key sort / typing / encode / K1 + K2 / emit run there); records that path does not model
    (nested objects, lists, multi-word strings, escapes, ...) are consolidated by the native host path (H1: C++ parse /
    alignment pre-pass / encode / decode + K1/K2/K4) inside the same call, and what that declines too (a key mixing objects
    with other types, string pairs that need the embeddings service, non-ASCII text, ...) takes the Python + GPU path."""
    from .. import _native
    if token_logprobs is not None:
        import contextlib
        import torch
        with torch.cuda.device(device) if torch.cuda.is_available() else contextlib.nullcontext():
            return _consolidate_weighted_batch(records, token_logprobs, consensus_settings, get_openai_embeddings_from_text, client,
                                               device, counts)
    default_eps = (consensus_settings.rel_eps, consensus_settings.abs_eps)
    native: List[Any] = [None] * len(records)
    if _native_settings(consensus_settings):
        by_n: dict = {}
        for i, texts in enumerate(records):
            if len(texts) >= 2:
                by_n.setdefault(len(texts), []).append(i)
        for n, idxs in by_n.items():
            _check_candidates(n)
            outs = _native_consolidate([records[i] for i in idxs], default_eps[0], default_eps[1], device)
            for i, o in zip(idxs, outs):
                native[i] = o
    results = []
    embed = get_openai_embeddings_from_text if get_openai_embeddings_from_text is not None else (lambda texts: [[0.0] for _ in texts])
    for texts, nat in zip(records, native):
        if nat is not None:
            results.append((nat[0], json.loads(nat[1])))
            continue
        contents = [_safe_parse_content(t) for t in texts if t]
        _check_candidates(len(contents))
        if len(texts) == 1:  # a single choice is returned as it is (reference consolidation.py:85-87)
            results.append((texts[0], None))
            continue
        # one non-empty content among several choices still goes through consensus_values, like the per-request path
        value, likelihoods = _consensus_sync(contents, consensus_settings, embed, client)
        results.append((_format_consensus_content(value), likelihoods))
    return results


def _consolidate_weighted_batch(records, token_logprobs, settings, embed_fn, client, device=0, counts=None):
    """consolidate_contents_batch with likelihood-weighted votes.  The token logprobs of every record's candidates (its non-empty
    texts, in order) are checked, then summed by ONE K3 launch.  With the default settings the records go to the weighted device
    JSON path (kc_consolidate_json_packed_weighted, one call per candidate count); what it declines, and every record under other
    settings, is aligned as the per-request path does (native pre-pass first) and consolidated by one weighted plan
    (consensus_values_batch)."""
    import numpy as np
    from .consensus_utils import consensus_values_batch
    if len(token_logprobs) != len(records):
        raise ValueError(f"token_logprobs has {len(token_logprobs)} records, records has {len(records)}")
    seqs, first = [], []  # first[r]: index of record r's first candidate sum
    for r, texts in enumerate(records):
        first.append(len(seqs))
        if len(texts) < 2:  # a single choice is returned as it is: its logprobs are not needed
            continue
        lps = token_logprobs[r]
        if lps is None or len(lps) != len(texts):
            raise ValueError(f"record {r}: token_logprobs needs one entry per candidate text ({len(texts)})")
        _check_candidates(sum(1 for t in texts if t))
        for c, t in enumerate(texts):
            if t:
                if lps[c] is None:
                    raise ValueError(f"vote weighting needs the token logprobs of every candidate; record {r}, candidate {c} has none")
                seqs.append(lps[c])
    flat, offsets = _pack_logprobs(seqs)
    sums = _logprob_sums(flat, offsets) if seqs else np.zeros(0, dtype=np.float32)
    results: List[Any] = [None] * len(records)
    if counts is not None:
        counts["device"] = 0
    if _native_settings(settings):
        by_n: dict = {}
        for r, texts in enumerate(records):
            m = sum(1 for t in texts if t)
            if len(texts) >= 2 and m >= 2:
                by_n.setdefault(m, []).append(r)
        for m, idxs in by_n.items():
            seq = np.concatenate([sums[first[r]:first[r] + m] for r in idxs])
            outs = _native_consolidate([[t for t in records[r] if t] for r in idxs], settings.rel_eps, settings.abs_eps, device,
                                       seq_logprobs=seq, counts=counts)
            for r, o in zip(idxs, outs):
                if o is not None:
                    results[r] = (o[0], json.loads(o[1]))
    embed = embed_fn if embed_fn is not None else (lambda texts: [[0.0] for _ in texts])
    todo, values, rows = [], [], []
    for r, texts in enumerate(records):
        if results[r] is not None:
            continue
        if len(texts) == 1:
            results[r] = (texts[0], None)
            continue
        contents = [_safe_parse_content(t) for t in texts if t]
        todo.append(r)
        values.append(_aligned_sync(contents, settings, embed, client))
        rows.append([float(x) for x in sums[first[r]:first[r] + len(contents)]])
    if todo:
        for r, (value, likelihoods) in zip(todo, consensus_values_batch(values, settings, embed, client, seq_logprobs=rows)):
            results[r] = (_format_consensus_content(value), likelihoods)
    return results
