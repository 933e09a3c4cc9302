"""Host logic of the native JSON path (H1: parse, key merge, planning, encoding, decoding, json.dumps formatting) on a machine
without a GPU: kc_json_plan -> the C oracle in the kernels' place -> kc_json_emit, against the reference's client order
(the object-level oracle).  The same generators as tests/test_gpu_json.py, where the real kernels sit in the middle."""
import random

from tests.helpers import consolidate_json_with_oracle
from tests.test_gpu_json import TEXT_EDGES, _expected, _random_nested_record, _random_record


def test_two_phase_native_json_matches_client_order_cpu():
    rng = random.Random(11)
    by_n = {}
    for _ in range(500):
        n = rng.choice([2, 3, 5, 8, 16])
        by_n.setdefault(n, []).append(_random_record(rng, n))
    for _ in range(300):
        n = rng.choice([2, 3, 5, 8])
        by_n.setdefault(n, []).append(_random_nested_record(rng, n))
    native = 0
    for _n, recs in by_n.items():
        for texts, got in zip(recs, consolidate_json_with_oracle(recs)):
            if got is None:
                continue
            native += 1
            assert got == _expected(texts), texts
    assert native > 600
    # string votes holding floats: the classes are sanitize_value(str(v)), so NaN / Infinity / -0.0 / 1e16 must be spelled
    # as str(float) spells them ("nan", "inf", "-0.0", "1e+16"), not as json.dumps does
    specials = [['{"s": "inf"}', '{"s": Infinity}', '{"s": -Infinity}', '{"s": NaN}'],
                ['{"s": "nan"}', '{"s": NaN}', '{"s": "x"}', '{"s": Infinity}'],
                ['{"s": "00"}', '{"s": -0.0}', '{"s": 1e16}', '{"s": -0.0}'],
                ['{"s": "1e16"}', '{"s": 1e16}', '{"s": -0.0}', '{"s": 1e16}']]
    for texts, got in zip(specials, consolidate_json_with_oracle(specials)):
        assert got is not None and got == _expected(texts), texts
    for texts, got in zip(TEXT_EDGES, consolidate_json_with_oracle(TEXT_EDGES)):
        assert got is not None and got == _expected(texts), texts


def test_two_phase_native_json_list_records_cpu():
    """Records with list fields through the native path (H2 alignment, then the plan of the aligned texts with an
    element-wise merge), the oracle in the kernels' place: the reference's client-order goldens, random list records and
    list records with escaped keys."""
    import json

    from oracle.gen_golden import random_list_records
    from tests.helpers import load_golden
    from tests.test_gpu_json import _expected_with_lists
    from k_llms_b200.utils.consolidation import _format_consensus_content
    by_n, native = {}, 0
    for case in load_golden("client_order"):
        if len(case["values"]) >= 2:
            by_n.setdefault(len(case["values"]), []).append(([json.dumps(v) for v in case["values"]], case))
    for _n, items in by_n.items():
        for (texts, case), got in zip(items, consolidate_json_with_oracle([t for t, _ in items])):
            assert got is not None, texts
            native += 1
            assert got == (_format_consensus_content(case["value"]), json.dumps(case["conf"])), (texts, got)
    assert native > 100
    recs = [[json.dumps(v) for v in r] for r in random_list_records(78, 200)]
    by_n = {}
    for r in recs:
        by_n.setdefault(len(r), []).append(r)
    for _n, rs in by_n.items():
        for texts, got in zip(rs, consolidate_json_with_oracle(rs)):
            assert got is not None and got == _expected_with_lists(texts), texts
    # escaped keys inside list elements and objects: decoded keys decide the order and the special-key skip
    keys = ["\reasoning___x", "x\"source___", "reasoning___q", 'q"', "q#", "q\\", "q\n", "Q"]
    rng = random.Random(5)
    recs = []
    for _ in range(60):
        n = rng.choice([2, 3])
        recs.append([json.dumps({"items": [{k: rng.choice([1, 2, None]) for k in rng.sample(keys, 3)} for _ in range(rng.randrange(1, 3))],
                                 "o": {k: rng.choice(["a", "b"]) for k in rng.sample(keys, 3)}}) for _ in range(n)])
    by_n = {}
    for r in recs:
        by_n.setdefault(len(r), []).append(r)
    for _n, rs in by_n.items():
        for texts, got in zip(rs, consolidate_json_with_oracle(rs)):
            assert got is not None and got == _expected_with_lists(texts), texts


def test_per_request_client_path_goes_native_cpu(monkeypatch):
    """consolidate_chat_completions / consolidate_parsed_chat_completions route a request through H1 (default settings): same
    consensus message, likelihoods and parsed object as the reference's client order — here with the oracle in the kernels'
    place; other settings and requests without an embeddings callable keep the Python path."""
    import json

    from openai.types.chat import ChatCompletion, ParsedChatCompletion
    from pydantic import BaseModel

    from k_llms_b200 import _native as K
    from k_llms_b200.utils import consolidation as C
    from k_llms_b200.utils.consensus_utils import ConsensusSettings
    from oracle.gen_golden import random_list_records
    from tests.helpers import raising_embeddings
    from tests.test_gpu_json import _expected_with_lists

    calls = []

    def fake_consolidate_json(records, *a, **k):
        calls.append(len(records))
        return consolidate_json_with_oracle(records)

    monkeypatch.setattr(C, "_native_consolidate", fake_consolidate_json)  # the seam in front of kc_consolidate_json_packed

    def completion_of(texts, cls=ChatCompletion):
        return cls.model_validate({"id": "x", "object": "chat.completion", "created": 0, "model": "m",
                                   "choices": [{"index": i, "finish_reason": "stop", "message": {"role": "assistant", "content": t}}
                                               for i, t in enumerate(texts)]})

    payloads = [{"name": "John", "age": 30, "active": True, "city": "Paris", "tags": ["a", "b"]},
                {"name": "John", "age": 30, "active": True, "city": "paris", "tags": ["b", "a"]},
                {"name": "Jon", "age": 31, "active": False, "city": "Paris", "tags": ["a", "b", "c"]}]
    cases = [[json.dumps(p) for p in payloads], ["Yes", "yes", "No"], ["the big cat sat", "the big cat sat", "a big cat sat"]]
    cases += [[json.dumps(v) for v in r] for r in random_list_records(5, 60)]
    for texts in cases:
        out = C.consolidate_chat_completions(completion_of(texts), raising_embeddings, client=None)
        exp_content, exp_lik = _expected_with_lists(texts)
        assert out.choices[0].message.content == exp_content and json.dumps(out.likelihoods) == exp_lik, texts
        assert [c.message.content for c in out.choices[1:]] == texts
    assert len(calls) == len(cases)

    class Person(BaseModel):
        name: str
        age: float
        active: bool
        city: str
        tags: list

    out = C.consolidate_parsed_chat_completions(completion_of(cases[0], ParsedChatCompletion), raising_embeddings, None,
                                                response_format=Person)
    assert out.choices[0].message.parsed == Person(name="John", age=30.0, active=True, city="Paris", tags=["a", "b"])
    # non-default settings and a missing embeddings callable do not take the native route
    n_calls = len(calls)
    assert C._consensus_of_choices_native(completion_of(cases[0]).choices, ConsensusSettings(min_support_ratio=0.6), raising_embeddings) is None
    assert C._consensus_of_choices_native(completion_of(cases[0]).choices, ConsensusSettings(), None) is None
    assert len(calls) == n_calls


def test_two_phase_native_json_mutated_texts_cpu():
    """Candidate texts with random byte edits (broken JSON, stray tokens, escapes, non-ASCII): whatever the native path
    accepts must equal the reference's client order; the rest it must decline."""
    import json

    from oracle.gen_golden import _record_candidates, random_list_records
    from tests.test_gpu_json import _expected_with_lists
    rng = random.Random(7)
    alphabet = '{}[]",:0123456789.eE-+ntf \\n\\t\\\\u00e9abcxyz'

    def mutate(text):
        chars = list(text)
        for _ in range(rng.randrange(1, 4)):
            if not chars:
                break
            i, r = rng.randrange(len(chars)), rng.random()
            if r < 0.4:
                chars[i] = rng.choice(alphabet)
            elif r < 0.7:
                del chars[i]
            else:
                chars.insert(i, rng.choice(alphabet))
        return "".join(chars)

    src = [[json.dumps(v) for v in r] for r in random_list_records(21, 150)]
    src += [[json.dumps(x) for x in _record_candidates(rng, rng.choice([2, 3, 5]), depth=2)] for _ in range(100)]
    by_n = {}
    for texts in src:
        texts = [mutate(t) if rng.random() < 0.4 else t for t in texts]
        if all(texts):
            by_n.setdefault(len(texts), []).append(texts)
    native = 0
    for _n, rs in by_n.items():
        for texts, got in zip(rs, consolidate_json_with_oracle(rs)):
            if got is not None:
                native += 1
                assert got == _expected_with_lists(texts), texts
    assert native > 150
