"""The device JSON path with KC_JSON_UNICODE (k_llms_b200/csrc/kc_jsoncore.cuh, kc_jsongpu.cuh) on a machine without a GPU:
similarity-medoid fields whose values hold non-ASCII text or \\uXXXX escapes stay on the device.  The host instantiation of the
phases (tests.helpers.jsongpu_with_oracle) must reproduce the reference's goldens byte for byte (tools/gen_golden_unicode.py),
decline what it does not model with a stable reason, print every code point as json.dumps does, and count words as str.split()
does.  Without the flag nothing changes."""
import ctypes as c
import json
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from oracle import consensus_py as O
from tests import weighted_oracle as W
from tests.helpers import MUTATE_ALPHABET, jsongpu_with_oracle, load_golden
from tests.test_async_native_host_logic import oracle_kernels, python_async  # noqa: F401  (a fixture)
from tests.test_gpu_json import _expected
from tests.test_weighted_host_logic import EMBED
from tools.gen_golden_unicode import PY_SPACES, enc_str, unicode_records

UNI = K.JSON_UNICODE | K.JSON_KEY_UNION
D_SYNTAX, D_ESCAPE_OR_NON_ASCII, D_KEYS_DIFFER, D_ALIGN = 2, 3, 7, 15


def goldens_by_n(reshaped=None):
    by_n = {}
    for case in load_golden("unicode_medoid"):
        if reshaped is None or case["reshaped"] == reshaped:
            by_n.setdefault(len(case["texts"]), []).append(case)
    return by_n


@pytest.mark.parametrize("flags", [UNI, K.JSON_UNICODE, UNI | K.JSON_LISTS], ids=["key_union", "same_shape", "lists"])
def test_goldens_byte_for_byte(flags):
    count = 0
    for _n, cases in goldens_by_n(None if flags & K.JSON_KEY_UNION else False).items():
        pairs, status = jsongpu_with_oracle([cs["texts"] for cs in cases], flags=flags)
        for cs, got, st in zip(cases, pairs, status):
            assert st == 0, (cs["texts"], st)
            assert got == (cs["content"], cs["likelihoods"]), cs["texts"]
            count += 1
    assert count >= (26 if flags & K.JSON_KEY_UNION else 20), count


def generated_by_n(seed, count, ns=(2, 3, 5, 8, 16, 33)):
    """The goldens' generator without the reference: records at more candidate counts, some with keys reordered or dropped.
    A record whose every member of a string field is under 3 words is a vote with non-ASCII text and declines."""
    by_n = {}
    for texts in unicode_records(seed, count, ns, reshape=True):
        by_n.setdefault(len(texts), []).append(texts)
    return by_n


def test_generated_records_match_the_client_order():
    accepted = 0
    for _n, recs in generated_by_n(21, 600).items():
        pairs, status = jsongpu_with_oracle(recs, flags=UNI)
        for texts, got, st in zip(recs, pairs, status):
            if st:
                assert st == D_ESCAPE_OR_NON_ASCII, (texts, st)
                continue
            accepted += 1
            assert got == _expected(texts), texts
    assert accepted > 500, accepted


def test_under_the_async_medoid(oracle_kernels):  # noqa: F811
    recs_by_n = generated_by_n(22, 200, ns=(2, 3, 5, 8))
    for n, cases in goldens_by_n().items():
        recs_by_n.setdefault(n, []).extend(cs["texts"] for cs in cases)
    accepted = 0
    for _n, recs in recs_by_n.items():
        pairs, status = jsongpu_with_oracle(recs, flags=UNI | K.JSON_NUMERIC_MEDOID)
        for texts, got, st in zip(recs, pairs, status):
            if st:
                assert st == D_ESCAPE_OR_NON_ASCII, (texts, st)
                continue
            accepted += 1
            assert got == python_async(texts), texts
    assert accepted > 150, accepted


def test_weighted():
    rng = np.random.default_rng(11)
    recs_by_n = generated_by_n(23, 300)
    for n, cases in goldens_by_n().items():
        recs_by_n.setdefault(n, []).extend(cs["texts"] for cs in cases)
    for n, recs in recs_by_n.items():
        seq = (-rng.exponential(4.0, len(recs) * n)).astype(np.float32)
        pairs, status = jsongpu_with_oracle(recs, seq, flags=UNI)
        for r, (texts, got, st) in enumerate(zip(recs, pairs, status)):
            if st:
                assert st == D_ESCAPE_OR_NON_ASCII, (texts, st)
                continue
            value, conf = W.client_order([json.loads(t) for t in texts], seq[r * n:(r + 1) * n], O.DEFAULTS, EMBED)
            assert got == (json.dumps(value), json.dumps(conf)), texts


def test_without_the_flag_every_golden_declines_as_before():
    for _n, cases in goldens_by_n().items():
        recs = [cs["texts"] for cs in cases]
        for flags in (0, K.JSON_KEY_UNION, K.JSON_KEY_UNION | K.JSON_LISTS):
            pairs, status = jsongpu_with_oracle(recs, flags=flags)
            assert all(p is None for p in pairs) and set(status) == {D_ESCAPE_OR_NON_ASCII}, (flags, status)


def plan_status(records, flags):
    """The device phases' statuses for candidate texts given as BYTES (invalid UTF-8 included)."""
    lib = K.load()
    n = len(records[0])
    enc = [t for r in records for t in r]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in enc], out=off[1:])
    blob = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8).copy()
    h = c.c_void_p()
    K.check(lib.kc_debug_jsongpu_plan_flags(blob.ctypes.data, off.ctypes.data, len(records), n, flags, c.byref(h)))
    try:
        vc, nc, st = c.c_void_p(), c.c_void_p(), c.c_void_p()
        gv, gx = c.c_int64(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_inputs(h, c.byref(vc), c.byref(gv), c.byref(nc), c.byref(gx), c.byref(st)))
        return [int(s) for s in np.ctypeslib.as_array(c.cast(st, c.POINTER(c.c_uint8)), shape=(len(records),))]
    finally:
        lib.kc_debug_jsongpu_free(h)


PHRASE = "café au lait please"
DECLINED = {
    # vote fields: every member has < 3 words, their classes need unidecode
    "vote_raw": ([{"a": "café"}, {"a": "cafe"}], D_ESCAPE_OR_NON_ASCII),
    "vote_escape_to_ascii": (['{"a": "\\u0041"}', '{"a": "A"}'], D_ESCAPE_OR_NON_ASCII),
    "vote_single_live": ([{"a": "été"}, {"a": None}], D_ESCAPE_OR_NON_ASCII),
    "key_raw": ([{"é": PHRASE}, {"é": PHRASE}], D_ESCAPE_OR_NON_ASCII),
    "key_escaped": (['{"\\u0061": "x y z"}', '{"a": "x y z"}'], D_ESCAPE_OR_NON_ASCII),
    "key_del": (['{"a\x7f": "x y z"}', '{"a\x7f": "x y z"}'], D_ESCAPE_OR_NON_ASCII),
    "bad_u_escape_short": (['{"a": "x y \\u12"}', '{"a": "x y z"}'], D_SYNTAX),
    "bad_u_escape_hex": (['{"a": "x y \\u12g4"}', '{"a": "x y z"}'], D_SYNTAX),
    "bad_u_escape_at_end": (['{"a": "x y \\u', '{"a": "x y z"}'], D_SYNTAX),
}
BAD_UTF8 = {
    "stray_continuation": b"\x80", "overlong_2": b"\xc0\xaf", "overlong_c1": b"\xc1\xbf", "overlong_3": b"\xe0\x80\xaf",
    "overlong_4": b"\xf0\x80\x80\xaf", "surrogate": b"\xed\xa0\x80", "surrogate_low": b"\xed\xbf\xbf", "above_10ffff": b"\xf4\x90\x80\x80",
    "f5_lead": b"\xf5\x80\x80\x80", "ff": b"\xff", "truncated_2": b"\xc3", "truncated_3": b"\xe2\x82", "truncated_4": b"\xf0\x9f\x98",
    "bad_second": b"\xc3\x28", "bad_third": b"\xe2\x82\x28",
}


def _texts(cands):
    return [t if isinstance(t, str) else json.dumps(t, ensure_ascii=False) for t in cands]


@pytest.mark.parametrize("name", sorted(DECLINED))
def test_declines(name):
    cands, why = DECLINED[name]
    _pairs, status = jsongpu_with_oracle([_texts(cands)], flags=UNI)
    assert status == [why], status


@pytest.mark.parametrize("name", sorted(BAD_UTF8))
def test_invalid_utf8_declines(name):
    bad = b'{"a": "one two ' + BAD_UTF8[name] + b' three"}'
    assert plan_status([[bad, b'{"a": "one two three"}']], UNI) == [D_ESCAPE_OR_NON_ASCII]
    assert plan_status([[b'{"a": "one two \xe2\x82\xac three"}', b'{"a": "one two three"}']], UNI) == [0]  # the euro sign is valid


def test_list_records_with_non_ascii_text_stay_declined():
    recs = [_texts([{"a": [PHRASE, "x"]}, {"a": [PHRASE]}]), _texts([{"a": PHRASE, "b": ["x"]}, {"a": PHRASE, "b": ["x"]}])]
    _pairs, status = jsongpu_with_oracle(recs, flags=UNI | K.JSON_LISTS)
    assert status == [D_ALIGN, D_ALIGN], status


def test_a_medoid_field_next_to_a_declined_vote_field_declines_the_record():
    recs = [_texts([{"a": PHRASE, "b": "é"}, {"a": PHRASE, "b": "e"}])]
    _pairs, status = jsongpu_with_oracle(recs, flags=UNI)
    assert status == [D_ESCAPE_OR_NON_ASCII]


def _random_code_points(rng, k):
    out = []
    for _ in range(k):
        r = rng.random()
        if r < 0.3:
            out.append(chr(rng.randrange(0x20, 0x7F)))
        elif r < 0.4:
            out.append(chr(rng.randrange(0, 0x20)) if rng.random() < 0.8 else "\x7f")
        elif r < 0.7:
            out.append(chr(rng.randrange(0x80, 0x10000)))
        else:
            out.append(chr(rng.randrange(0x10000, 0x110000)))
    return "".join(out)


def test_printer_matches_json_dumps_over_all_planes():
    """A lone multi-word string is its own consensus: its printed form must be json.dumps of what json.loads reads."""
    rng = random.Random(5)
    recs, want = [], []
    for _ in range(3000):
        s = "w1 w2 w3 " + _random_code_points(rng, rng.randrange(1, 40))
        text = '{"a": ' + enc_str(rng, s) + "}"
        recs.append([text, '{"a": null}'])
        want.append(json.dumps({"a": json.loads(text)["a"]}))
    pairs, status = jsongpu_with_oracle(recs, flags=UNI)
    for text, got, st, w in zip(recs, pairs, status, want):
        assert st == 0 and got[0] == w, (text, got, w)


def test_word_count_is_str_split():
    """A lone non-ASCII string is a medoid (kept) with >= 3 words of str.split(), else a vote (declined)."""
    rng = random.Random(9)
    pieces = ["a", "é", "b1", "東", "\U0001f600", ""]
    recs, multi = [], []
    for _ in range(4000):
        parts = [rng.choice(pieces) for _ in range(rng.randrange(1, 6))]
        s = "é"
        for p in parts:
            s += rng.choice(PY_SPACES + [" ", " ", "\u200b", "\u2060", "-", ""]) + p
        recs.append(['{"a": ' + enc_str(rng, s) + "}", '{"a": null}'])
        multi.append(len(s.split()) >= 3)
    _pairs, status = jsongpu_with_oracle(recs, flags=UNI)
    for r, m, st in zip(recs, multi, status):
        assert st == (0 if m else D_ESCAPE_OR_NON_ASCII), (r, m, st)
    assert 1000 < sum(multi) < 3000


def test_mutated_records_never_give_a_wrong_answer():
    """Byte-level mutations of the goldens and of generated records (multi-byte characters and escapes in the alphabet): what
    the device path accepts equals the oracle's client order."""
    rng = random.Random(13)
    alphabet = list(MUTATE_ALPHABET) + ["é", "€", "\U0001f600", "\\u00e9", "\\uD83D\\uDE00", "\\ud800", "\u00a0", "\u3000", "\\u000b"]
    accepted = 0
    recs_by_n = generated_by_n(24, 800, ns=(2, 3, 5, 8))
    for n, cases in goldens_by_n().items():
        recs_by_n.setdefault(n, []).extend(cs["texts"] for cs in cases)
    for n, originals in recs_by_n.items():
        recs = []
        for orig in originals:
            texts = []
            for t in orig:
                chars = list(t)
                for _ in range(rng.randrange(1, 3)):
                    i, r = rng.randrange(len(chars)), rng.random()
                    if r < 0.4:
                        chars[i] = rng.choice(alphabet)
                    elif r < 0.7:
                        del chars[i]
                    else:
                        chars.insert(i, rng.choice(alphabet))
                texts.append("".join(chars) if rng.random() < 0.5 else t)
            recs.append(texts)
        pairs, status = jsongpu_with_oracle(recs, flags=UNI)
        for texts, got, st in zip(recs, pairs, status):
            if st:
                continue
            accepted += 1
            assert got == _expected(texts), texts
    assert accepted > 150, accepted
