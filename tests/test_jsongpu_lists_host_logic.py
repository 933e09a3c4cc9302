"""The device JSON path's list round (KC_JSON_LISTS, k_llms_b200/csrc/kc_jsongpu.cuh) on a machine without a GPU: records with list
fields are marked by the first round, aligned by the native pre-pass H2 on the host, and consolidated from the aligned texts with
list nodes.  The host instantiation of the phases (kc_debug_jsongpu_plan_flags with KC_JSON_LISTS) runs both rounds lane by lane
with the oracle in the kernels' place; its texts must equal the reference's client-order goldens, the host path H1 (which
consolidates from the aligned texts too) and the Python pre-pass + oracle, byte for byte.  Without the flag nothing changes."""
import json
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from oracle import consensus_py as O
from tests import weighted_oracle as W
from tests.helpers import consolidate_json_with_oracle, jsongpu_with_oracle, load_golden
from tests.test_async_native_host_logic import oracle_kernels, python_async  # noqa: F401  (a fixture)
from tests.test_gpu_json import _expected, _expected_with_lists
from tests.test_weighted_host_logic import EMBED
from tools.jsonpacked_throughput import invoice_lines_texts

LISTS = K.JSON_KEY_UNION | K.JSON_LISTS
D_NESTED, D_NUMBER_RANGE, D_ALIGN = 4, 12, 15


def list_records(seed, count):
    """Random list records of every generator, grouped by candidate count (2 ... 64)."""
    from oracle.gen_golden import _record_candidates, random_list_records
    rng = random.Random(seed)
    recs = [[json.dumps(v) for v in r] for r in random_list_records(seed, count)]
    for _ in range(count // 2):
        recs.append([json.dumps(c) for c in _record_candidates(rng, rng.choice([2, 3, 5, 8, 16, 33, 64]), depth=3)])
    for n in (2, 3, 8, 16, 64):
        recs.extend(invoice_lines_texts(count // 20, n, seed + n))
    by_n = {}
    for r in recs:
        by_n.setdefault(len(r), []).append(r)
    return by_n


def _has_list(texts):
    return any("[" in t for t in texts)


def _declined_as_expected(texts, why, host=False):
    """The generators' records the device path leaves to the host: numbers outside the exact conversion range, empty objects,
    and (host: H1 declines them too) a list or an object against None after the alignment."""
    return why == D_NUMBER_RANGE or (why in (D_NESTED, 13) and (host or any("{}" in t for t in texts)))


def test_reference_goldens_on_the_device_path():
    from k_llms_b200.utils.consolidation import _format_consensus_content
    by_n = {}
    for case in load_golden("client_order"):
        if len(case["values"]) >= 2:
            by_n.setdefault(len(case["values"]), []).append(([json.dumps(v) for v in case["values"]], case))
    on_device = with_lists = 0
    for _n, items in by_n.items():
        pairs, status = jsongpu_with_oracle([t for t, _ in items], flags=LISTS)
        for (texts, case), got, st in zip(items, pairs, status):
            assert st == 0, (texts, st)  # every golden stays on the device
            on_device += 1
            with_lists += _has_list(texts)
            assert got == (_format_consensus_content(case["value"]), json.dumps(case["conf"])), (texts, got)
    assert on_device >= 125 and with_lists >= 120, (on_device, with_lists)


def test_async_goldens_on_the_device_path():
    """The reference's async client order (async_recursive_list_alignments + async_consensus_values) on records with lists."""
    from k_llms_b200.utils.consolidation import _format_consensus_content
    accepted = 0
    declined = {}
    for case in load_golden("async_cases"):
        texts = [json.dumps(v) for v in case["values"]]
        if case["kind"] != "client_order" or len(texts) < 2 or not _has_list(texts):
            continue
        (got,), (st,) = jsongpu_with_oracle([texts], flags=LISTS | K.JSON_NUMERIC_MEDOID)
        if st:
            declined[st] = declined.get(st, 0) + 1
            continue
        accepted += 1
        assert got == (_format_consensus_content(case["value"]), json.dumps(case["conf"])), (texts, got)
    # 11: a numeric element holding strings or bools too (the async medoid compares them by its own rules)
    assert accepted >= 50 and set(declined) <= {11, D_NUMBER_RANGE}, (accepted, declined)


def test_random_list_records_match_the_host_path_and_the_python_pre_pass():
    on_device = 0
    for n, recs in list_records(31, 500).items():
        pairs, status = jsongpu_with_oracle(recs, flags=LISTS)
        host = consolidate_json_with_oracle(recs)
        for texts, got, st, h1 in zip(recs, pairs, status, host):
            if st:
                assert _declined_as_expected(texts, st, host=h1 is None), (texts, st)
                continue
            on_device += 1
            assert got == h1, texts  # re-serialising the aligned values changes no byte
            if n <= 16:
                assert got == _expected_with_lists(texts), texts
    assert on_device > 600, on_device


def test_weighted_list_records():
    from k_llms_b200.utils.consensus_utils import recursive_list_alignments
    rng = np.random.default_rng(11)
    for n, recs in list_records(47, 200).items():
        if n > 16:
            continue
        seq = (-rng.exponential(4.0, len(recs) * n)).astype(np.float32)
        pairs, status = jsongpu_with_oracle(recs, seq, flags=LISTS)
        for r, (texts, got, st) in enumerate(zip(recs, pairs, status)):
            if st:
                assert _declined_as_expected(texts, st, host=True), (texts, st)
                continue
            contents = [json.loads(t) for t in texts]
            aligned, _ = recursive_list_alignments(contents, "embeddings", EMBED, None, 0.51)
            value, conf = W.client_order(contents, seq[r * n:(r + 1) * n], O.DEFAULTS, EMBED, aligned=aligned)
            assert got == (json.dumps(value), json.dumps(conf)), (texts, got)


def test_async_list_records_match_the_python_async_route(oracle_kernels):  # noqa: F811
    on_device = 0
    for n, recs in list_records(53, 200).items():
        if n > 16:
            continue
        pairs, status = jsongpu_with_oracle(recs, flags=LISTS | K.JSON_NUMERIC_MEDOID)
        for texts, got, st in zip(recs, pairs, status):
            if st:
                assert st == 11 or _declined_as_expected(texts, st, host=True), (texts, st)  # 11: numbers mixed with strings / bools
                continue
            on_device += 1
            assert got == python_async(texts), texts
    assert on_device > 150, on_device


EDGES = {
    "object against a list": (['{"a": {"b": 1}}', '{"a": [1]}'], D_NESTED),
    "list against a scalar": (['{"a": [1, 2]}', '{"a": 3}'], 7),  # the aligned round: another token count
    "an empty object in a list": (['{"a": [{}]}', '{"a": [{}]}'], D_NESTED),
    "a special key in an element": (['{"a": [{"reasoning___x": 1, "v": 2}]}', '{"a": [{"reasoning___x": 1, "v": 2}]}'], 9),
    "two long strings in an element": (['{"a": ["' + "word " * 12 + '"]}', '{"a": ["' + "other " * 12 + '"]}'], D_ALIGN),
    "more than 8 levels through lists": (['{"a": ' + "[" * 9 + "1" + "]" * 9 + "}"] * 2, D_NESTED),
    "non-ASCII in an element": (['{"a": ["café"]}', '{"a": ["cafe"]}'], 3),
    "an empty candidate": (['{"a": [1]}', ""], 13),
    "an escape in a list": (['{"a": ["\\u00e9"]}', '{"a": ["e"]}'], 3),
    "free text": (['{"a": [1]}', "not json"], 1),
}


@pytest.mark.parametrize("name", sorted(EDGES))
def test_declined_with_a_stable_reason(name):
    texts, why = EDGES[name]
    (got,), (st,) = jsongpu_with_oracle([texts], flags=LISTS)
    assert got is None and st == why, (texts, st)
    # the same in a batch, whatever comes before it
    pairs, status = jsongpu_with_oracle([['{"k": 1}', '{"k": 2}'], texts, ['{"x": [1, 2]}', '{"x": [2, 1]}']], flags=LISTS)
    assert status[1] == why and pairs[1] is None and status[0] == 0 and status[2] == 0


def test_accepted_edges():
    cases = [
        ['{"a": []}', '{"a": []}'],
        ['{"a": [[1, 2], [3]], "b": "x"}', '{"a": [[1, 2], [3]], "b": "y"}', '{"a": [[1, 2], [3]], "b": "x"}'],
        ['{"a": [null, {"b": 1}]}', '{"a": [null, {"b": 2}]}'],
        ['{"z": [{"y": true, "x": "q"}], "a": {"l": [1.5, 2]}}', '{"a": {"l": [1.5, 2]}, "z": [{"x": "Q", "y": true}]}'],
        ['{"a": ' + "[" * 8 + "1" + "]" * 8 + "}"] * 3,
    ]
    for texts in cases:
        (got,), (st,) = jsongpu_with_oracle([texts], flags=LISTS)
        assert st == 0, (texts, st)
        assert got == _expected_with_lists(texts), texts


def test_mixed_batches_agree_and_without_the_flag_nothing_changes():
    from tests.test_jsongpu_union_host_logic import union_record
    rng = random.Random(3)
    recs = []
    lists = list_records(61, 100)[3]
    for i in range(len(lists)):
        recs.append(lists[i])
        recs.append(union_record(rng, 3))
    with_flag, st_flag = jsongpu_with_oracle(recs, flags=LISTS)
    without, st_without = jsongpu_with_oracle(recs, flags=K.JSON_KEY_UNION)
    for texts, a, sa, b, sb in zip(recs, with_flag, st_flag, without, st_without):
        alone, (st_alone,) = jsongpu_with_oracle([texts], flags=LISTS)
        assert (a, sa) == (alone[0], st_alone), texts
        if _has_list(texts):
            assert sb == D_NESTED and b is None, (texts, sb)
        else:
            assert (a, sa) == (b, sb), texts
            if sa == 0:
                assert a == _expected(texts), texts
