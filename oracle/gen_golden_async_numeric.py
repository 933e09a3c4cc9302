"""Golden vectors of the reference's ASYNC numeric medoid (TEST INFRASTRUCTURE; run in the build container, where the reference
exists):  python -m oracle.gen_golden_async_numeric  ->  tests/golden/async_numeric.json

The reference's async dispatcher has no numeric clustering (consensus_utils.py:1638-1688): a number that is not an enum-like
vote takes the similarity medoid (numerical_similarity, np.nanmean of each row, first argmax), and the result is the ORIGINAL
object.  Two kinds of case:
  "group"   one field's values (n = 2..64): ulp ties between rows with the same close-count, values exactly 1 % apart, +-0,
            int / float spellings of one value, 19-digit ints, Nones.  Recorded: async_consensus_values' (value, conf); the
            value's type matters (20 and 20.0 are equal, but print apart).
  "texts"   candidate JSON texts of one shape, flat or nested, with numbers spelled as the texts spell them ("20", "20.0",
            "2e1", "-0"): the async client order (async_recursive_list_alignments, then async_consensus_values) and the texts
            the product returns (json.dumps of the value and of the likelihoods)."""
from __future__ import annotations

import asyncio
import json
import logging
import os
import random

from oracle.gen_golden import GOLDEN_DIR
from oracle.ref_loader import load_reference


async def _raising(texts):
    raise RuntimeError("network embeddings are not available in the oracle")


FIXED_GROUPS = [
    [10, 10, 20, 20], [10, 10, 20, 20, 30], [20, 20.0, 20], [20.0, 20, 20], [0, -0.0, 0.0], [-0.0, 0, 5], [100, 101, 102],
    [100, 99, 101, 98], [1.0, 1.01, 1.02], [1234567890123456789, 1234567890123456788, 1234567890123456789, 1240000000000000000],
    [None, 7, None], [None, 3.5, 3.5, None, 4], [1e-300, 0, -1e-300], [1, 2, 3, 4, 5, 6, 7, 8, 9],
]


def _value_pool(rng: random.Random, style: str):
    if style == "classes":  # few classes: rows tie on their close-count
        base = rng.choice([1, 10, 100, 1000])
        return [base * m for m in rng.sample([1, 2, 3, 5, 7], rng.randint(2, 5))]
    if style == "edge":  # exactly 1 % apart, on both sides
        b = rng.choice([100, 200, 1000, 1.0, 2.5])
        return [b, b * 1.01, b * 0.99, b + b / 100, b - b / 100, b * 1.02]
    if style == "zeros":
        return [0, -0.0, 0.0, 1e-300, -5e-324, 1]
    if style == "spellings":
        v = rng.choice([20, 3, 1000])
        return [v, float(v), v + 1]
    if style == "bigint":
        b = rng.randrange(10 ** 18, 10 ** 19)
        return [b, b + 1, b + 10 ** 17, int(b * 1.005)]
    return [rng.uniform(-1e3, 1e3) for _ in range(4)]  # "random"


STYLES = ("classes", "edge", "zeros", "spellings", "bigint", "random")


def random_groups(seed: int):
    rng = random.Random(seed)
    groups = []
    for n in range(2, 65):
        for style in STYLES:
            pool = _value_pool(rng, style)
            p_none = rng.choice([0.0, 0.0, 0.2])
            groups.append([None if rng.random() < p_none else rng.choice(pool) for _ in range(n)])
    return groups


def _spell(v, rng: random.Random) -> str:
    """One JSON spelling of the number v (None -> null)."""
    if v is None:
        return "null"
    if isinstance(v, float) and v == int(v) and abs(v) < 1e15 and rng.random() < 0.3:
        return f"{int(v)}e0" if v else rng.choice(["0.0", "-0.0"])
    if isinstance(v, int) and v == 0 and rng.random() < 0.3:
        return "-0"
    return json.dumps(v)


def text_records(seed: int):
    rng = random.Random(seed)
    records = [
        [json.dumps({"v": 10}), json.dumps({"v": 10}), json.dumps({"v": 20}), json.dumps({"v": 20})],
        ['{"v": 20}', '{"v": 20.0}', '{"v": 2e1}'],
        ['{"v": 2e1}', '{"v": 20}', '{"v": 20.0}'],
        ['{"v": -0}', '{"v": 0.0}', '{"v": -0.0}'],
        ['{"a": 1, "b": {"x": 10, "y": "k"}}', '{"a": 1.0, "b": {"x": 10.0, "y": "k"}}', '{"a": 2, "b": {"x": 11, "y": "j"}}'],
    ]
    for n in (2, 3, 5, 8, 16, 33, 64):
        for _ in range(6):
            nested = rng.random() < 0.5
            pools = {f: _value_pool(rng, rng.choice(STYLES)) for f in ("n0", "n1", "n2")}
            cands = []
            for _c in range(n):
                fields = []
                for f, pool in pools.items():
                    v = None if rng.random() < 0.1 else rng.choice(pool)
                    fields.append(f'"{f}": {_spell(v, rng)}')
                fields.append(f'"s": "{rng.choice(["alpha", "beta"])}"')
                fields.append(f'"t": {rng.choice(["true", "false"])}')
                body = ", ".join(fields)
                if nested:
                    v = rng.choice(pools["n0"])
                    body = f'"inner": {{"m": {_spell(v, rng)}, "w": "x"}}, ' + body
                cands.append("{" + body + "}")
            records.append(cands)
    return records


def main() -> None:
    logging.disable(logging.CRITICAL)
    cu = load_reference()
    settings = cu.ConsensusSettings()

    async def consensus(vals):
        return await cu.async_consensus_values(vals, settings, _raising, client=None)

    async def client_order(vals):
        aligned, _ = await cu.async_recursive_list_alignments(vals, settings.string_similarity_method, _raising, None, settings.min_support_ratio)
        aligned = [(d if isinstance(d, dict) else {}) for d in aligned]
        return await cu.async_consensus_values(aligned, settings, _raising, client=None)

    cases = []
    for vals in FIXED_GROUPS + random_groups(424242):
        v, c = asyncio.run(consensus(vals))
        cases.append({"kind": "group", "values": vals, "value": v, "conf": c})
    for texts in text_records(777):
        v, c = asyncio.run(client_order([json.loads(t) for t in texts]))
        cases.append({"kind": "texts", "texts": texts, "content": json.dumps(v), "likelihoods": json.dumps(c)})
    meta = {"generator": "oracle/gen_golden_async_numeric.py", "reference": "retab-dev/k-LLMs @ 089dba9 behind 3 import stubs",
            "entry": "async_consensus_values / async_recursive_list_alignments with a raising embeddings coroutine"}
    with open(os.path.join(GOLDEN_DIR, "async_numeric.json"), "w") as f:
        json.dump({"meta": meta, "cases": cases}, f, separators=(",", ":"))
    print(f"wrote async_numeric.json: {len(cases)} cases")


if __name__ == "__main__":
    main()
