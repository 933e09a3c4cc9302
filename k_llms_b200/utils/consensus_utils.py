"""Drop-in for `k_llms.utils.consensus_utils` — the seven names `consolidation.py` imports
(reference consolidation.py:11-19) — with the scalar-field consensus on the GPU.

`consensus_values` keeps the reference signature and return shape (consensus_utils.py:1376-1382, "cu"):
the recursion over dicts and lists is planned on the host (k_llms_b200.columnar), every str/bool vote
(cu:936-982) and every numeric clustering (cu:1098-1219) of the record runs in ONE launch each of the sm_100a
kernels behind `libkllms_b200.so`, and the result tree is rebuilt.  `consensus_values_batch` is the new batched
entry (many records per launch) the reference lacks.

There is NO CPU implementation of the hot path here: without the CUDA library or a device these functions raise.
"""
from __future__ import annotations

import asyncio
import logging
import warnings
from typing import Any, Awaitable, Callable, List, Literal, Optional, Sequence, Tuple

from pydantic import BaseModel

from .. import columnar
from . import similarity

logger = logging.getLogger(__name__)

StringSimilarityMethod = Literal["levenshtein", "jaccard", "hamming", "embeddings"]
StringConsensusMethod = Literal["centroid", "llm-consensus"]
SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE = Callable[[List[str]], List[List[float]]]
ASYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE = Callable[[List[str]], Awaitable[List[List[float]]]]


class ConsensusSettings(BaseModel):
    """Same fields and defaults as the reference model (cu:53-69).  Only allow_none_as_candidate,
    string_similarity_method, string_consensus_method, min_support_ratio, rel_eps and abs_eps are read by
    the reference's code paths; the others are accepted for compatibility."""

    allow_none_as_candidate: bool = False
    string_similarity_method: StringSimilarityMethod = "embeddings"
    string_consensus_method: StringConsensusMethod = "centroid"
    minimum_voters_threshold: float = 0.75
    min_support_ratio: float = 0.51
    rel_eps: float = 0.03
    abs_eps: float = 1e-6
    base_maj_thresh: float = 0.6
    maj_loosen_k: float = 0.1
    trim_frac: float = 0.2


def _host_primitive(settings: ConsensusSettings):
    def run(values: list, parent_valid_frac: float, embed):
        if isinstance(values[0], str) and settings.string_consensus_method == "llm-consensus" \
                and settings.string_similarity_method == "embeddings":
            # cu:1090-1096 asks gpt-5-mini for a consensus string: a network call, outside this build's scope
            raise NotImplementedError("string_consensus_method='llm-consensus' needs a network LLM call; use 'centroid'")
        return similarity.medoid(values, settings.string_similarity_method, embed, parent_valid_frac)
    return run


def _plan_for(n: int, settings: ConsensusSettings, numeric_branch: bool = True, weighted: bool = False) -> columnar.Plan:
    plan = columnar.Plan(n, settings.allow_none_as_candidate, settings.rel_eps, settings.abs_eps, _host_primitive(settings),
                         numeric_branch=numeric_branch, weighted=weighted)
    plan.string_method = settings.string_similarity_method if settings.string_consensus_method == "centroid" else "host"
    return plan


def _record_sums(seq: Sequence[float], n_values: int, where: str) -> List[float]:
    """The sequence logprobs of one record's candidates, checked: one number per candidate, finite as float32 (extra entries of
    a padded row are ignored)."""
    import numpy as np
    if len(seq) < n_values:
        raise ValueError(f"{where}: {len(seq)} sequence logprobs for {n_values} candidates")
    with np.errstate(over="ignore"):  # a sum beyond the float32 range becomes inf and is refused below
        out = np.asarray([float(s) for s in list(seq)[:n_values]], dtype=np.float64).astype(np.float32)
    if not np.isfinite(out).all():  # checked as the kernel sees them: float32
        raise ValueError(f"{where}: sequence logprobs must be finite as float32, got {list(seq)[:n_values]}")
    return [float(s) for s in out]


def consensus_values(
    values: List[Any],
    consensus_settings: ConsensusSettings,
    sync_get_openai_embeddings_from_text: SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    parent_valid_frac: float = 1.0,
    _numeric_branch: bool = True,
    seq_logprobs: Optional[Sequence[float]] = None,
) -> Tuple[Any, Any]:
    """(consensus value, confidence) for one record's n candidate values — cu:1376-1454.  seq_logprobs (n floats, the
    candidates' summed token logprobs): the vote leaves are likelihood-weighted (DESIGN.md §5)."""
    weighted = seq_logprobs is not None
    sums = _record_sums(seq_logprobs, len(values), "consensus_values") if weighted else None
    plan = _plan_for(len(values), consensus_settings, _numeric_branch, weighted)
    if weighted:
        plan.begin_record(sums)
    root = plan.add(values, parent_valid_frac, sync_get_openai_embeddings_from_text)
    res = plan.run() if (plan.vote_rows or plan.num_rows or plan.medoid_groups) else {}
    return plan.materialise(root, res)


def consensus_values_batch(
    records: Sequence[List[Any]],
    consensus_settings: Optional[ConsensusSettings] = None,
    sync_get_openai_embeddings_from_text: Optional[SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE] = None,
    client: Any = None,
    parent_valid_frac: float = 1.0,
    seq_logprobs: Optional[Any] = None,
) -> List[Tuple[Any, Any]]:
    """Batched entry (new): consensus_values for many independent records with ONE K1 and ONE K2 launch.

    seq_logprobs: float32 [R][n] (n >= every record's candidate count; row r's first len(records[r]) entries are record r's
    candidate sums, e.g. from K3): the vote leaves are likelihood-weighted (DESIGN.md §5), with ONE K3b launch for the batch."""
    settings = consensus_settings or ConsensusSettings()
    embed = sync_get_openai_embeddings_from_text if sync_get_openai_embeddings_from_text is not None else _no_embeddings
    weighted = seq_logprobs is not None
    if weighted:
        if len(seq_logprobs) != len(records):
            raise ValueError(f"consensus_values_batch: {len(seq_logprobs)} rows of sequence logprobs for {len(records)} records")
        sums = [_record_sums(s, len(values), f"consensus_values_batch, record {r}")
                for r, (values, s) in enumerate(zip(records, seq_logprobs))]
    plan = _plan_for(max((len(r) for r in records), default=1), settings, weighted=weighted)
    roots = []
    for r, values in enumerate(records):
        if weighted:
            plan.begin_record(sums[r])
        roots.append(plan.add(values, parent_valid_frac, embed))
    res = plan.run() if (plan.vote_rows or plan.num_rows or plan.medoid_groups) else {}
    return [plan.materialise(root, res) for root in roots]


def _no_embeddings(texts):
    raise RuntimeError("no embeddings callable was supplied")  # the similarity code then falls back to Levenshtein


async def async_consensus_values(
    values: List[Any],
    consensus_settings: ConsensusSettings,
    async_get_openai_embeddings_from_text: ASYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    parent_valid_frac: float = 1.0,
    seq_logprobs: Optional[Sequence[float]] = None,
) -> Tuple[Any, Any]:
    """Async twin (cu:1779-1860).  The reference's async primitive has NO numeric clustering (cu:1638-1688, SURVEY.md §0.5):
    a non-unanimous numeric field takes the similarity medoid — [10, 10, 11] gives (10, 0.5) here and (10.0, 0.66667) in the
    sync path.  That difference is part of the reference's behaviour and is reproduced; votes still run on the GPU, off the
    event loop.  seq_logprobs: as for consensus_values."""
    loop = asyncio.get_running_loop()

    def embed(texts):
        fut = asyncio.run_coroutine_threadsafe(async_get_openai_embeddings_from_text(texts), loop)
        return fut.result()

    return await asyncio.to_thread(consensus_values, values, consensus_settings,
                                   embed if async_get_openai_embeddings_from_text is not None else None, client,
                                   parent_valid_frac, False, seq_logprobs)


# ----------------------------------------------------------------------------- alignment pre-pass


def recursive_list_alignments(
    values: List[Any],
    string_similarity_method: StringSimilarityMethod,
    sync_get_openai_embeddings_from_text: SYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    min_support_ratio: float,
    max_novelty_ratio: float = 0.25,
    current_path: str = "",
    reference_idx: Optional[int] = None,
):
    """The pre-pass `consolidation.py` runs before the vote (cu:458-613).

    Dict payloads: every candidate gets every key, keys sorted, missing -> None, recursively (cu:516-548) — this is
    what flat records need and it is implemented here.  Lists are aligned by the separate module
    `k_llms_b200.utils.list_alignment` (reference cu:185-430 + majority_sorting.py)."""
    from copy import deepcopy
    if not values:
        return values, {}
    if all(v is None for v in values):
        return values, {current_path: [current_path for _ in values]}
    non_nulls = [v for v in values if v is not None]
    values = deepcopy(values)  # cu:504
    first_type = type(non_nulls[0])
    same_type = all(isinstance(x, first_type) for x in non_nulls)
    key_mappings: dict = {}
    if not same_type or first_type not in (dict, list):
        key_mappings[current_path] = [current_path if (v is not None or idx == reference_idx) else None
                                      for idx, v in enumerate(values)]
        return values, key_mappings
    if first_type is dict:
        dicts_only = [(d if isinstance(d, dict) else {}) for d in values]
        all_keys = sorted({k for d in dicts_only for k in d})
        for key in all_keys:
            sub_path = f"{current_path}.{key}" if current_path else key
            aligned, sub_map = recursive_list_alignments(
                [d.get(key) for d in dicts_only], string_similarity_method, sync_get_openai_embeddings_from_text, client,
                min_support_ratio, max_novelty_ratio=max_novelty_ratio, current_path=sub_path, reference_idx=reference_idx)
            for d, v in zip(dicts_only, aligned):
                d[key] = v
            key_mappings.update(sub_map)
        return [{k: d.get(k) for k in all_keys} for d in dicts_only], key_mappings
    from .list_alignment import align_list_values
    return align_list_values(values, string_similarity_method, sync_get_openai_embeddings_from_text, client, min_support_ratio,
                             max_novelty_ratio, current_path, reference_idx, recursive_list_alignments)


async def async_recursive_list_alignments(
    values: List[Any],
    string_similarity_method: StringSimilarityMethod,
    async_get_openai_embeddings_from_text: ASYNC_GET_OPENAI_EMBEDDINGS_FROM_TEXT_TYPE,
    client: Any,
    min_support_ratio: float,
    max_novelty_ratio: float = 0.25,
    current_path: str = "",
    reference_idx: Optional[int] = None,
):
    loop = asyncio.get_running_loop()

    def embed(texts):
        return asyncio.run_coroutine_threadsafe(async_get_openai_embeddings_from_text(texts), loop).result()

    return await asyncio.to_thread(recursive_list_alignments, values, string_similarity_method, embed, client,
                                   min_support_ratio, max_novelty_ratio, current_path, reference_idx)
