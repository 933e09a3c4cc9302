"""Golden vectors for the device JSON path's non-ASCII similarity medoids (KC_JSON_UNICODE).  Run where the reference is
installed:  python -m tools.gen_golden_unicode  ->  tests/golden/unicode_medoid.json

Each record has ASCII vote, bool and numeric fields next to multi-word string fields whose candidate TEXTS hold non-ASCII text
written every way JSON allows: raw UTF-8 and \\uXXXX escapes in either hex case (Latin-1, curly quotes, dashes, the euro sign,
CJK-only words), astral characters raw and as surrogate-pair escapes, lone surrogate escapes, escapes that decode to ASCII
letters, quotes, backslashes and control characters, and words separated by each of Python's 29 whitespace code points (or
joined by zero-width characters that are not whitespace), so that the word count decides vote against medoid.  A `note` field
holds strings of 45-55 code points whose UTF-8 is longer than 50 bytes.

The texts are written here, byte by byte, because json.dumps would choose one spelling.  The reference decides each record
through its client order (ref_loader.ref_client_order); its consensus and likelihoods are stored as json.dumps prints them.
The set is kept small (a few dozen records at n = 2 and 3); the tests draw many more records from the same generator and
compare them with the oracle's port of the client order (oracle/consensus_py.py).  The reference's unidecode stub asserts ASCII input and only vote fields reach it, so a record
that reaches it is drawn again: every golden is a record whose non-ASCII text is decided by the similarity medoid alone.

`unicode_records` (no reference needed) generates more records of the same kind."""
from __future__ import annotations

import json
import os
import random

PY_SPACES = [chr(c) for c in range(0x110000) if chr(c).isspace()]  # the 29 separators of str.split()
JOINERS = ["\u200b", "\u2060", "\u200d", "\ufeff"]  # zero-width, not whitespace: they join two words

WORDS = ("invoice total payment bank transfer goods services street road avenue suite floor office delivery "
         "parcel express contact customer account").split()
UNI_WORDS = ["café", "Zürich", "São", "Paulo", "naïve", "Ærø", "Straße", "façade", "Müller", "Ñandú", "crème", "brûlée",
             "“quoted”", "‘single’", "it’s", "—", "–", "€100", "£5", "½", "…", "東京", "日本語", "北京市", "株式会社",
             "😀", "🚚", "📦✓", "🇫🇷", "\u212amart", "İstanbul", "ﬁle", "２０２４", "Ω", "\u00a0x", "x\u0085"]
ODD_WORDS = ['say "hi"', "back\\slash", "a/b", "\x01ctl", "tab\tbed", "line\nfeed", "del\x7f", "\x1fus", "bell\x07",
             "\ud800lone", "lone\udfff", "\udbff", "ABC", "Zz9"]


def _hex(rng, v):
    return ("\\u%04x" if rng.random() < 0.5 else "\\u%04X") % v


def enc_str(rng, s):
    """A JSON string literal for s, each character spelled raw or escaped at random (every spelling json.loads reads as s)."""
    out = ['"']
    two = {'"': '\\"', "\\": "\\\\", "\n": "\\n", "\r": "\\r", "\t": "\\t", "\b": "\\b", "\f": "\\f"}
    for ch in s:
        c = ord(ch)
        r = rng.random()
        if ch in two:
            out.append(two[ch] if r < 0.7 else _hex(rng, c))
        elif c < 0x20 or 0xD800 <= c <= 0xDFFF:
            out.append(_hex(rng, c))
        elif c < 0x80:
            out.append(("\\/" if ch == "/" else _hex(rng, c)) if r < 0.08 else ch)
        elif c >= 0x10000:
            v = c - 0x10000
            out.append(ch if r < 0.5 else _hex(rng, 0xD800 + (v >> 10)) + _hex(rng, 0xDC00 + (v & 0x3FF)))
        else:
            out.append(ch if r < 0.6 else _hex(rng, c))
    out.append('"')
    return "".join(out)


TEXT_KEYS = ("description", "name", "note")  # the multi-word fields; keys and the other fields are plain ASCII


def enc(rng, v, key=None):
    if isinstance(v, dict):
        return "{" + ", ".join(json.dumps(k) + ": " + enc(rng, x, k) for k, x in v.items()) + "}"
    if isinstance(v, str) and key in TEXT_KEYS:
        return enc_str(rng, v)
    return json.dumps(v)


def _sep(rng):
    r = rng.random()
    if r < 0.7:
        return " "
    if r < 0.9:
        return rng.choice(PY_SPACES)
    return rng.choice(JOINERS)


def phrase(rng, k):
    pool = rng.random()
    words = []
    for _ in range(k):
        r = rng.random()
        words.append(rng.choice(UNI_WORDS) if r < 0.45 + 0.3 * pool else (rng.choice(ODD_WORDS) if r < 0.6 + 0.3 * pool else rng.choice(WORDS)))
    out = words[0]
    for w in words[1:]:
        out += _sep(rng) + w
    return out


def _noisy(rng, s):
    r = rng.random()
    if r < 0.4:
        return s
    words = s.split(" ")
    if r < 0.6 and len(words) > 1:
        words.pop(rng.randrange(len(words)))
    elif r < 0.8:
        words[rng.randrange(len(words))] = rng.choice(UNI_WORDS + WORDS)
    elif r < 0.9:
        words.append(rng.choice(UNI_WORDS))
    else:
        return s.upper()
    return " ".join(words)


def _sized(rng, L):
    """A string of exactly L code points, rich in multi-byte characters."""
    s = phrase(rng, 12)
    while len(s) < L:
        s += " " + phrase(rng, 4)
    return s[:L]


def record_values(rng, n):
    """n candidate objects around one truth (Python values)."""
    truth = {"id": rng.randrange(1000), "status": rng.choice(["paid", "open", "overdue", "void"]),
             "total": round(rng.uniform(1, 5000), 2), "urgent": rng.random() < 0.5,
             "description": phrase(rng, rng.randrange(3, 9)),
             "vendor": {"name": phrase(rng, rng.randrange(3, 6)), "country": rng.choice(["FR", "DE", "JP", "BR"])}}
    with_note = rng.random() < 0.5
    cands = []
    for c in range(n):
        d = {"id": truth["id"] if rng.random() < 0.8 else rng.randrange(1000),
             "status": truth["status"] if rng.random() < 0.7 else rng.choice(["Paid", "open", "OPEN", "void"]),
             "total": truth["total"] if rng.random() < 0.7 else round(truth["total"] * rng.uniform(0.9, 1.1), 2),
             "urgent": truth["urgent"] if rng.random() < 0.8 else None,
             "description": _noisy(rng, truth["description"]) if rng.random() < 0.92 else None,
             "vendor": {"name": _noisy(rng, truth["vendor"]["name"]), "country": truth["vendor"]["country"]}}
        if with_note:  # one member may pass 50 code points, the others stay at or under it (K4's contract)
            d["note"] = _sized(rng, rng.randrange(45, 56) if c == 0 else rng.randrange(45, 51))
        cands.append(d)
    return cands


def texts_of(rng, cands, reshape):
    """Candidate texts; with `reshape` some candidates reorder their keys or drop one."""
    out = []
    for d in cands:
        if reshape and rng.random() < 0.4:
            items = list(d.items())
            rng.shuffle(items)
            if rng.random() < 0.3:
                items.pop(rng.randrange(len(items)))
            d = dict(items)
        out.append(enc(rng, d))
    return out


def _normalize(s):
    return "".join(ch for ch in s if ch.isascii() and ch.isalnum()).lower()


def in_contract(texts):
    """K4's rule for every multi-word group: at most one string over 50 code points, one normalised string over 64."""
    vals = [json.loads(t) for t in texts]

    def leaves(v, path=()):
        for k, x in v.items():
            if isinstance(x, dict):
                yield from leaves(x, path + (k,))
            else:
                yield path + (k,), x
    groups = {}
    for v in vals:
        for p, x in leaves(v):
            groups.setdefault(p, []).append(x)
    for xs in groups.values():
        ss = [x for x in xs if isinstance(x, str)]
        if any(len(s.split()) >= 3 for s in ss) and (sum(len(s) > 50 for s in ss) > 1 or sum(len(_normalize(s)) > 64 for s in ss) > 1):
            return False
    return True


def unicode_records(seed, count, ns=(2, 3, 5, 8, 16), reshape=False):
    """count records of candidate texts, in K4's contract (some may still hold a vote field with non-ASCII text)."""
    rng = random.Random(seed)
    out = []
    while len(out) < count:
        texts = texts_of(rng, record_values(rng, rng.choice(ns)), reshape)
        if in_contract(texts):
            out.append(texts)
    return out


def main() -> None:
    import logging

    from oracle.gen_golden import GOLDEN_DIR
    from oracle.ref_loader import ref_client_order
    logging.disable(logging.CRITICAL)
    cases, drawn = [], 0
    for reshape, seed, count in ((False, 2718, 20), (True, 3141, 6)):
        rng = random.Random(seed)
        got = 0
        while got < count:
            drawn += 1
            texts = texts_of(rng, record_values(rng, rng.choice((2, 3))), reshape)
            if not in_contract(texts):
                continue
            vals = [json.loads(t) for t in texts]
            try:
                value, conf = ref_client_order(vals)
            except AssertionError:  # a vote field with non-ASCII text reached the unidecode stub
                continue
            cases.append({"texts": texts, "reshaped": reshape, "content": json.dumps(value), "likelihoods": json.dumps(conf)})
            got += 1
    meta = {"generator": "tools/gen_golden_unicode.py", "reference": "retab-dev/k-LLMs @ 089dba9 behind 3 import stubs",
            "entry": "ref_client_order with raising embeddings"}
    with open(os.path.join(GOLDEN_DIR, "unicode_medoid.json"), "w", encoding="utf-8") as f:
        f.write('{"meta":' + json.dumps(meta) + ',"cases":[\n')  # one case per line
        f.write(",\n".join(json.dumps(cs, separators=(",", ":"), ensure_ascii=False) for cs in cases) + "\n]}\n")
    print(f"wrote unicode_medoid.json: {len(cases)} cases ({drawn} drawn)")


if __name__ == "__main__":
    main()
