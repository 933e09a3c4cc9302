// kc_jsoncore.cuh — the per-thread building blocks of the device JSON path (H1g): a validating scanner for flat JSON objects,
// exact decimal -> float64 and float64 -> float.__repr__ conversions, sanitised string comparison.
//
// Everything here is __host__ __device__ and free of warp intrinsics: the kernels in kc_jsongpu.cuh call these functions
// per lane, and the CPU tests instantiate THE SAME code on the host (kc_debug_jsongpu_* in kllms_b200.cu) to check the logic
// against the oracle in a container without a GPU.  What each piece replaces in the reference:
//     scan_object      json.loads of one candidate content (consolidation.py:25-38) for objects of scalar values
//     to_double        float(text) / float(int(text)) as json.loads + consensus_utils.py:1105-1114 produce them (correctly rounded)
//     sanitized_equal  sanitize_value(a) == sanitize_value(b)  (consensus_utils.py:925-933, ASCII)
//     float_repr       json.dumps of a float = float.__repr__ (shortest round-trip digits, Ryu), _format_consensus_content
//                      (consolidation.py:41-60); the host path H1 (kc_json.cpp) prints its floats through it as well
#pragma once

#include <stdint.h>
#include <string.h>

#include "kc_internal.h"  // KC_HD
#include "kc_ryu_tables.cuh"

namespace kc {
namespace js {

typedef unsigned __int128 u128;

// value kinds of a token (JSON scalar types; nested values and non-standard tokens make the scanner decline)
// K_OPEN / K_CLOSE: a nested object's `"key": {` and its `}` — structure tokens between which the object's members follow;
// K_LOPEN / K_LCLOSE: a list's `"key": [` and its `]` (only when the scanner is asked for list nodes), its elements between them
enum : uint8_t { K_NULL = 0, K_TRUE = 1, K_FALSE = 2, K_INT = 3, K_FLOAT = 4, K_STR = 5, K_OPEN = 6, K_CLOSE = 7, K_LOPEN = 8, K_LCLOSE = 9 };
KC_HD inline bool is_open(uint32_t k) { return k == K_OPEN || k == K_LOPEN; }
KC_HD inline bool is_close(uint32_t k) { return k == K_CLOSE || k == K_LCLOSE; }
// which kernel decides a field (plan_leaf in kc_json.cpp; consensus_utils.py:1405-1411 vote, :1443-1453 numeric)
// F_MEDOID: a string field that is not enum-like (some value has >= 3 words): the similarity medoid, K4 (:1221-1237)
enum : uint8_t { F_ALLNULL = 0, F_VOTE_STR = 1, F_VOTE_BOOL = 2, F_NUMERIC = 3, F_MEDOID = 4, F_OPEN = 5, F_CLOSE = 6, F_LOPEN = 7, F_LCLOSE = 8 };
constexpr int32_t kMaxNesting = 8;  // nested objects and lists below the top level; the depth lives in the token's flags (4 bits)

// One (field, candidate) cell of a record: views into the chunk's text.  Strings: the raw inner span (no quotes); raw == value
// unless TOK_ESCAPED (keys: always, the scanner declines escapes in keys).  flags: bit 0 TOK_MULTIWORD, bit 1 TOK_ESCAPED, bit 2
// TOK_ELEM, bit 3 TOK_UNICODE, bits 4-7 the nesting depth of the member.  K_OPEN / K_LOPEN carry the key of the nested value,
// K_CLOSE / K_LCLOSE no key.  TOK_MULTIWORD: the string has >= 3 whitespace-separated words (not enum-like, cu:1405).  TOK_ELEM:
// a list element (no key).
struct alignas(16) Tok {
    uint32_t vstart, vlen;  // value span, relative to the chunk's first byte
    uint32_t kstart;        // key span (inner)
    uint16_t klen;
    uint8_t kind;
    uint8_t flags;
};
constexpr uint8_t TOK_MULTIWORD = 1;
KC_HD inline uint32_t tok_depth(const Tok &t) { return (uint32_t)t.flags >> 4; }  // 0 = a member of the top-level object
constexpr uint8_t TOK_ESCAPED = 2;  // the span holds escapes: two-character ones (\" \\ \/ \b \f \n \r \t), \uXXXX only with TOK_UNICODE
constexpr uint8_t TOK_ELEM = 4;
// a string value (scanned with `unicode`) that holds raw UTF-8, a \uXXXX escape or a raw DEL: its readers decode it to code
// points (decode_cp) instead of reading bytes
constexpr uint8_t TOK_UNICODE = 8;

// why a record left the device path (diagnostics only; every non-zero code means "host path").  D_ALIGN: the alignment
// pre-pass of the list round declined the record (a pair of long strings for the embeddings service, non-ASCII text).
enum : int32_t {
    D_OK = 0, D_NOT_OBJECT = 1, D_SYNTAX = 2, D_ESCAPE_OR_NON_ASCII = 3, D_NESTED = 4, D_NONSTANDARD_NUMBER = 5, D_TOO_MANY_FIELDS = 6,
    D_KEYS_DIFFER = 7, D_DUP_KEY = 8, D_SPECIAL_KEY = 9, D_MULTIWORD = 10, D_MIXED_TYPES = 11, D_NUMBER_RANGE = 12, D_EMPTY = 13,
    D_TOO_LONG = 14, D_ALIGN = 15,
};

KC_HD inline bool is_json_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
KC_HD inline bool is_digit(uint8_t c) { return (uint8_t)(c - '0') <= 9; }

// str.isspace() of a code point: the 29 separators str.split() splits on
KC_HD inline bool is_py_space(uint32_t c) {
    if (c < 0x80) return c == ' ' || (c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x1F);
    return c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) || c == 0x2028 || c == 0x2029 || c == 0x202F ||
           c == 0x205F || c == 0x3000;
}

// the four hex digits of a \uXXXX escape (either case); false if one is not a hex digit
KC_HD inline bool hex4(const uint8_t *s, uint32_t &v) {
    v = 0;
    for (int k = 0; k < 4; ++k) {
        const uint8_t c = s[k];
        uint32_t d;
        if (is_digit(c)) d = (uint32_t)(c - '0');
        else if ((c | 32) >= 'a' && (c | 32) <= 'f') d = (uint32_t)((c | 32) - 'a' + 10);
        else return false;
        v = (v << 4) | d;
    }
    return true;
}

// One UTF-8 sequence at s[0..avail) (s[0] >= 0x80) as Python's strict decoder reads it: its length, 0 when it is invalid
// (a stray continuation byte, an overlong form, an encoded surrogate ED A0..BF, a code point above U+10FFFF, a truncated sequence)
KC_HD inline uint32_t utf8_decode(const uint8_t *s, uint32_t avail, uint32_t &cp) {
    const uint8_t b = s[0];
    if (b < 0xC2 || b > 0xF4) return 0;
    const uint32_t k = b < 0xE0 ? 2u : (b < 0xF0 ? 3u : 4u);
    if (avail < k) return 0;
    // the second byte's range excludes overlong forms (E0, F0), surrogates (ED) and code points above U+10FFFF (F4)
    const uint8_t lo = b == 0xE0 ? 0xA0 : (b == 0xF0 ? 0x90 : 0x80), hi = b == 0xED ? 0x9F : (b == 0xF4 ? 0x8F : 0xBF);
    if (s[1] < lo || s[1] > hi) return 0;
    cp = b & (0x7Fu >> k);
    for (uint32_t i = 1; i < k; ++i) {
        if ((s[i] & 0xC0) != 0x80) return 0;
        cp = (cp << 6) | (s[i] & 0x3Fu);
    }
    return k;
}

KC_HD inline int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

KC_HD inline uint64_t f64_bits(double x) {
    uint64_t b;
    memcpy(&b, &x, 8);
    return b;
}
KC_HD inline double bits_f64(uint64_t b) {
    double x;
    memcpy(&x, &b, 8);
    return x;
}

// ---------------------------------------------------------------- scanner

// Scans ONE candidate text `s[0..len)` as json.loads would an object of scalars and nested objects.  Token j goes to
// toks[j * stride] when toks != nullptr (spans are stored relative to `rel`: s == chunk + rel); a nested object is its K_OPEN
// token, its members' tokens, its K_CLOSE token.  Returns the token count (>= 1) or -D_* — the scanner never guesses: whatever
// it does not model exactly (\u escapes, non-ASCII, lists, NaN/Infinity, free text that the reference wraps as {"text": ...},
// an empty object) is left to the host path.  *nested (optional): whether the object holds a nested object (or a list).
// lists: `[` opens a list node (K_LOPEN, its elements keyless TOK_ELEM tokens one level deeper, K_LCLOSE) instead of declining
// the record with D_NESTED; *has_list (optional): whether the text holds a list.  unicode: string VALUES may hold raw UTF-8
// (validated), \uXXXX escapes and a raw DEL (the token gets TOK_UNICODE, its words are counted over Python's whitespace) instead
// of declining the record with D_ESCAPE_OR_NON_ASCII; keys stay ASCII without DEL or escapes (json.dumps prints them as they are).
KC_HD inline int32_t scan_object(const uint8_t *s, uint32_t len, uint32_t rel, Tok *toks, int32_t stride, int32_t cap, bool *nested = nullptr,
                                 bool lists = false, bool *has_list = nullptr, bool unicode = false) {
    uint32_t p = 0;
    while (p < len && is_json_ws(s[p])) ++p;
    if (p >= len) return -D_EMPTY;
    if (s[p] != '{') return -D_NOT_OBJECT;
    ++p;
    while (p < len && is_json_ws(s[p])) ++p;
    if (p < len && s[p] == '}') return -D_EMPTY;  // {}: consensus of empty dicts — rare, host path
    int32_t j = 0;
    uint32_t depth = 0;
    uint32_t in_list = 0;  // bit d: the members of depth d are list elements
    if (nested) *nested = false;
    if (has_list) *has_list = false;
    for (;;) {
        while (p < len && is_json_ws(s[p])) ++p;
        const bool elem = (in_list >> depth) & 1u;
        Tok t;
        t.flags = 0;
        if (elem) {
            t.kstart = rel + p;
            t.klen = 0;
        } else {
            if (p >= len || s[p] != '"') return -D_SYNTAX;
            ++p;
            const uint32_t kstart = p;
            for (;;) {
                if (p >= len) return -D_SYNTAX;
                const uint8_t c = s[p];
                if (c == '"') break;
                if (c < 0x20) return -D_SYNTAX;
                if (c >= 0x7F || c == '\\') return -D_ESCAPE_OR_NON_ASCII;  // the emit prints a key's bytes: DEL and escapes decline
                ++p;
            }
            const uint32_t klen = p - kstart;
            if (klen > 0xFFFFu) return -D_TOO_LONG;
            ++p;
            while (p < len && is_json_ws(s[p])) ++p;
            if (p >= len || s[p] != ':') return -D_SYNTAX;
            ++p;
            while (p < len && is_json_ws(s[p])) ++p;
            t.kstart = rel + kstart;
            t.klen = (uint16_t)klen;
        }
        if (p >= len) return -D_SYNTAX;
        const uint8_t c = s[p];
        if (c == '"') {
            ++p;
            const uint32_t vs = p;
            uint32_t words = 0;
            bool prev_space = true;
            bool escaped = false, uni = false;
            for (;;) {
                if (p >= len) return -D_SYNTAX;
                const uint8_t d = s[p];
                if (d == '"') break;
                if (d < 0x20) return -D_SYNTAX;
                bool sp = d == ' ';  // the only ASCII str.split() whitespace a raw JSON string can hold unescaped
                if (d >= 0x7F) {
                    if (!unicode) return -D_ESCAPE_OR_NON_ASCII;
                    if (d > 0x7F) {
                        uint32_t cp = 0;
                        const uint32_t k = utf8_decode(s + p, len - p, cp);
                        if (k == 0) return -D_ESCAPE_OR_NON_ASCII;
                        sp = is_py_space(cp);
                        p += k - 1;
                    }
                    uni = true;  // DEL too: json.dumps prints it as \u007f
                } else if (d == '\\') {
                    // the two-character escapes stay in the token (TOK_ESCAPED; every reader of the value skips or maps them);
                    // \uXXXX (any code point, surrogate pairs, non-ASCII) is the host path's unless `unicode`
                    if (p + 1 >= len) return -D_SYNTAX;
                    const uint8_t e = s[p + 1];
                    if (e == 'u') {
                        if (!unicode) return -D_ESCAPE_OR_NON_ASCII;
                        uint32_t v;
                        if (p + 5 >= len || !hex4(s + p + 2, v)) return -D_SYNTAX;
                        sp = is_py_space(v);  // no surrogate is whitespace: a pair need not be joined to count words
                        uni = true;
                        p += 4;
                    } else {
                        if (!(e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't')) return -D_SYNTAX;
                        sp = e == 't' || e == 'n' || e == 'r' || e == 'f';  // str.split() whitespace; \b (0x08) is not
                    }
                    escaped = true;
                    ++p;
                }
                words += (!sp && prev_space) ? 1u : 0u;
                prev_space = sp;
                ++p;
            }
            t.kind = K_STR;
            t.vstart = rel + vs;
            t.vlen = p - vs;
            t.flags = (uint8_t)((words >= 3 ? TOK_MULTIWORD : 0) | (escaped ? TOK_ESCAPED : 0) | (uni ? TOK_UNICODE : 0));
            ++p;
        } else if (c == '{') {
            ++p;
            while (p < len && is_json_ws(s[p])) ++p;
            if (p < len && s[p] == '}') return -D_NESTED;              // an empty nested object: host path
            if ((int32_t)depth >= kMaxNesting) return -D_NESTED;
            t.kind = K_OPEN;
            t.vstart = rel + p;
            t.vlen = 0;
            t.flags = (uint8_t)((depth << 4) | (elem ? TOK_ELEM : 0));
            if (j >= cap) return -D_TOO_MANY_FIELDS;
            if (toks) toks[(int64_t)j * stride] = t;
            ++j;
            ++depth;
            in_list &= ~(1u << depth);
            if (nested) *nested = true;
            continue;  // the object's first member
        } else if (c == '[' && lists) {
            ++p;
            if ((int32_t)depth >= kMaxNesting) return -D_NESTED;
            if (has_list) *has_list = true;
            if (nested) *nested = true;
            t.kind = K_LOPEN;
            t.vstart = rel + p;
            t.vlen = 0;
            t.flags = (uint8_t)((depth << 4) | (elem ? TOK_ELEM : 0));
            if (j >= cap) return -D_TOO_MANY_FIELDS;
            if (toks) toks[(int64_t)j * stride] = t;
            ++j;
            while (p < len && is_json_ws(s[p])) ++p;
            if (p >= len || s[p] != ']') {
                ++depth;
                in_list |= 1u << depth;
                continue;  // the list's first element
            }
            ++p;  // [] : its K_LCLOSE follows at once, then whatever follows a value
            t.kind = K_LCLOSE;
            t.vstart = rel + p;
            t.kstart = rel + p;
            t.klen = 0;
            t.flags = (uint8_t)(depth << 4);
        } else if (c == 't') {
            if (len - p < 4 || s[p + 1] != 'r' || s[p + 2] != 'u' || s[p + 3] != 'e') return -D_SYNTAX;
            t.kind = K_TRUE;
            t.vstart = rel + p;
            t.vlen = 4;
            p += 4;
        } else if (c == 'f') {
            if (len - p < 5 || s[p + 1] != 'a' || s[p + 2] != 'l' || s[p + 3] != 's' || s[p + 4] != 'e') return -D_SYNTAX;
            t.kind = K_FALSE;
            t.vstart = rel + p;
            t.vlen = 5;
            p += 5;
        } else if (c == 'n') {
            if (len - p < 4 || s[p + 1] != 'u' || s[p + 2] != 'l' || s[p + 3] != 'l') return -D_SYNTAX;
            t.kind = K_NULL;
            t.vstart = rel + p;
            t.vlen = 4;
            p += 4;
        } else if (c == '-' || is_digit(c)) {
            const uint32_t vs = p;
            if (s[p] == '-') ++p;
            if (p >= len) return -D_SYNTAX;
            if (s[p] == '0') {
                ++p;
            } else if (s[p] >= '1' && s[p] <= '9') {
                while (p < len && is_digit(s[p])) ++p;
            } else {
                return s[p] == 'I' ? -D_NONSTANDARD_NUMBER : -D_SYNTAX;  // -Infinity
            }
            bool is_float = false;
            if (p < len && s[p] == '.') {
                ++p;
                if (p >= len || !is_digit(s[p])) return -D_SYNTAX;
                while (p < len && is_digit(s[p])) ++p;
                is_float = true;
            }
            if (p < len && (s[p] == 'e' || s[p] == 'E')) {
                ++p;
                if (p < len && (s[p] == '+' || s[p] == '-')) ++p;
                if (p >= len || !is_digit(s[p])) return -D_SYNTAX;
                while (p < len && is_digit(s[p])) ++p;
                is_float = true;
            }
            t.kind = is_float ? K_FLOAT : K_INT;
            t.vstart = rel + vs;
            t.vlen = p - vs;
        } else if (c == '[') {
            return -D_NESTED;  // lists need the alignment pre-pass: host path
        } else if (c == 'N' || c == 'I') {
            return -D_NONSTANDARD_NUMBER;  // NaN / Infinity: json.loads accepts them; the host path models them
        } else {
            return -D_SYNTAX;
        }
        if (t.kind != K_LCLOSE) t.flags = (uint8_t)(t.flags | (depth << 4) | (elem ? TOK_ELEM : 0));
        if (j >= cap) return -D_TOO_MANY_FIELDS;
        if (toks) toks[(int64_t)j * stride] = t;
        ++j;
        bool done = false;
        for (;;) {  // after a value: the next member, or the end of one or more objects / lists
            while (p < len && is_json_ws(s[p])) ++p;
            if (p >= len) return -D_SYNTAX;
            if (s[p] == ',') {
                ++p;
                break;
            }
            const bool closes_list = (in_list >> depth) & 1u;
            if (s[p] != (closes_list ? ']' : '}')) return -D_SYNTAX;
            ++p;
            if (depth == 0) {
                done = true;
                break;
            }
            --depth;
            Tok e;
            e.kind = closes_list ? K_LCLOSE : K_CLOSE;
            e.vstart = rel + p;
            e.vlen = 0;
            e.kstart = rel + p;
            e.klen = 0;
            e.flags = (uint8_t)(depth << 4);
            if (j >= cap) return -D_TOO_MANY_FIELDS;
            if (toks) toks[(int64_t)j * stride] = e;
            ++j;
        }
        if (done) break;
    }
    while (p < len && is_json_ws(s[p])) ++p;
    if (p != len) return -D_SYNTAX;
    return j;
}

// ---------------------------------------------------------------- strings

KC_HD inline bool is_alnum_lower(uint8_t &c) {  // lower-cases c; true if it survives sanitize_value's [^a-zA-Z0-9] filter
    if (c >= 'A' && c <= 'Z') c = (uint8_t)(c + 32);
    return (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9');
}

// sanitize_value(a) == sanitize_value(b) on ASCII text: lower-case, keep [a-z0-9] (consensus_utils.py:925-933)
// (a backslash in a value span always starts a two-character escape, and none of the escaped characters is alphanumeric:
// the pair is skipped as a whole — "\n" must not leave an 'n')
KC_HD inline bool sanitized_equal(const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb) {
    uint32_t i = 0, j = 0;
    for (;;) {
        uint8_t ca = 0, cb = 0;
        while (i < la) {
            ca = a[i];
            if (is_alnum_lower(ca)) break;
            i += ca == '\\' ? 2u : 1u;
        }
        while (j < lb) {
            cb = b[j];
            if (is_alnum_lower(cb)) break;
            j += cb == '\\' ? 2u : 1u;
        }
        if (i >= la || j >= lb) return i >= la && j >= lb;
        if (ca != cb) return false;
        ++i;
        ++j;
    }
}

// normalize_string(s) on ASCII text (consensus_utils.py:660-673: the same lower-case [a-z0-9] filter): its length, and the
// characters written to `out` (K4's input) when out != nullptr
KC_HD inline uint32_t sanitized_copy(const uint8_t *a, uint32_t la, uint8_t *out) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < la; ++i) {
        uint8_t c = a[i];
        if (!is_alnum_lower(c)) {
            i += c == '\\' ? 1u : 0u;
            continue;
        }
        if (out) out[k] = c;
        ++k;
    }
    return k;
}

// len(value) of a string token: every escape stands for one character
KC_HD inline uint32_t unescaped_length(const uint8_t *a, uint32_t la) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < la; ++i, ++k) i += a[i] == '\\' ? 1u : 0u;
    return k;
}

// The code point at a[i] of a TOK_UNICODE span (validated by scan_object), advancing i past it: what json.loads decodes.  A
// \uXXXX high surrogate followed by a \uXXXX low surrogate is one code point; any other surrogate escape stands alone.
KC_HD inline uint32_t decode_cp(const uint8_t *a, uint32_t la, uint32_t &i) {
    const uint8_t b = a[i];
    if (b == '\\') {
        const uint8_t e = a[i + 1];
        if (e != 'u') {
            i += 2;
            return e == 'b' ? 8u : (e == 'f' ? 12u : (e == 'n' ? 10u : (e == 'r' ? 13u : (e == 't' ? 9u : (uint32_t)e))));
        }
        uint32_t v, w;
        hex4(a + i + 2, v);
        i += 6;
        if (v >= 0xD800 && v < 0xDC00 && i + 6 <= la && a[i] == '\\' && a[i + 1] == 'u' && hex4(a + i + 2, w) && w >= 0xDC00 && w < 0xE000) {
            i += 6;
            return 0x10000u + ((v - 0xD800u) << 10) + (w - 0xDC00u);
        }
        return v;
    }
    if (b < 0x80) {
        ++i;
        return b;
    }
    uint32_t cp = 0;
    i += utf8_decode(a + i, la - i, cp);
    return cp;
}

// normalize_string (consensus_utils.py:660-673) of a TOK_UNICODE span: re.sub(r"[^a-zA-Z0-9]", "", text).lower() drops every
// non-ASCII code point before lower-casing (so the Kelvin sign and U+0130 leave nothing), keeps ASCII alphanumerics however they
// are written (A is 'A').  Its length, and the characters written to `out` (K4's input) when out != nullptr.
KC_HD inline uint32_t normalize_string(const uint8_t *a, uint32_t la, uint8_t *out) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < la;) {
        const uint32_t cp = decode_cp(a, la, i);
        uint8_t c = (uint8_t)cp;
        if (cp >= 0x80 || !is_alnum_lower(c)) continue;
        if (out) out[k] = c;
        ++k;
    }
    return k;
}

// len(value) of a TOK_UNICODE span: its code points
KC_HD inline uint32_t code_points(const uint8_t *a, uint32_t la) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < la; ++k) decode_cp(a, la, i);
    return k;
}

// bytewise three-way comparison (Python's str ordering on ASCII keys)
KC_HD inline int key_compare(const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb) {
    const uint32_t m = la < lb ? la : lb;
    for (uint32_t i = 0; i < m; ++i)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

KC_HD inline bool contains(const uint8_t *s, uint32_t len, const char *needle, uint32_t nl) {
    if (len < nl) return false;
    for (uint32_t i = 0; i + nl <= len; ++i) {
        uint32_t k = 0;
        while (k < nl && s[i + k] == (uint8_t)needle[k]) ++k;
        if (k == nl) return true;
    }
    return false;
}

// ---------------------------------------------------------------- decimal -> float64, exactly

// p * 2^exp2 (+ something strictly between 0 and one unit of p's last place when `sticky`) rounded to nearest-even.
// p != 0; the result is a normal double (callers guarantee the range).
KC_HD inline double u128_to_double(u128 p, bool sticky, int exp2) {
    const uint64_t hi = (uint64_t)(p >> 64), lo = (uint64_t)p;
    int msb = hi ? 127 - clz64(hi) : 63 - clz64(lo);
    uint64_t mant;
    if (msb <= 52) {
        mant = lo << (52 - msb);  // exact (callers never pass sticky here)
    } else {
        const int sh = msb - 52;
        mant = (uint64_t)(p >> sh);
        const u128 rem = p & ((((u128)1) << sh) - 1), half = ((u128)1) << (sh - 1);
        if (rem > half || (rem == half && (sticky || (mant & 1)))) {
            ++mant;
            if (mant == (1ull << 53)) {
                mant >>= 1;
                ++msb;
            }
        }
    }
    return bits_f64(((uint64_t)(msb + exp2 + 1023) << 52) | (mant & ((1ull << 52) - 1)));
}

// The float64 nearest to the JSON number s[0..len) (grammar already validated by scan_object): what float(json.loads(s))
// gives.  Exact integer arithmetic — no tables: up to 19 significant digits, |decimal exponent| <= 19 (22 for short mantissas).
// Returns false where that range is exceeded (the record goes to the host path, which uses strtod).
KC_HD inline bool to_double(const uint8_t *s, uint32_t len, double &out) {
    uint32_t p = 0;
    bool neg = false;
    if (p < len && s[p] == '-') {
        neg = true;
        ++p;
    }
    uint64_t w = 0;
    int sig = 0, frac = 0, dropped = 0;
    bool seen_dot = false;
    for (; p < len; ++p) {
        const uint8_t c = s[p];
        if (c == '.') {
            seen_dot = true;
            continue;
        }
        if (!is_digit(c)) break;
        if (sig < 19) {
            w = w * 10 + (uint64_t)(c - '0');
            if (w) ++sig;
            if (seen_dot) ++frac;
        } else {
            if (c != '0') return false;  // a 20th significant digit: not exactly representable in the 64-bit mantissa
            if (!seen_dot) ++dropped;    // trailing integer zeros scale the value
        }
    }
    int e10 = dropped - frac;
    if (p < len && (s[p] == 'e' || s[p] == 'E')) {
        ++p;
        bool eneg = false;
        if (p < len && (s[p] == '+' || s[p] == '-')) {
            eneg = s[p] == '-';
            ++p;
        }
        int ev = 0;
        for (; p < len; ++p) {
            if (ev > 9999) return false;
            ev = ev * 10 + (int)(s[p] - '0');
        }
        e10 += eneg ? -ev : ev;
    }
    double r;
    if (w == 0) {
        r = 0.0;
    } else if (e10 >= 0) {
        if (e10 > 19) return false;
        uint64_t p10 = 1;
        for (int i = 0; i < e10; ++i) p10 *= 10;
        r = u128_to_double((u128)w * p10, false, 0);
    } else {
        const int k = -e10;
        if (w <= (1ull << 53) && k <= 22) {  // both operands exact doubles: one correctly rounded division (Clinger)
            double d = 1.0;
            for (int i = 0; i < k; ++i) d *= 10.0;  // every partial product is exact up to 1e22
            r = (double)w / d;
        } else if (k <= 19) {
            uint64_t p10 = 1;
            for (int i = 0; i < k; ++i) p10 *= 10;
            const int sh = 64 + clz64(w);
            const u128 x = ((u128)w) << sh;  // top bit at position 127: the quotient keeps >= 63 significant bits
            const u128 q = x / p10;
            const bool sticky = (x - q * p10) != 0;
            r = u128_to_double(q, sticky, -sh);
        } else {
            return false;
        }
    }
    out = neg ? -r : r;
    return true;
}

// ---------------------------------------------------------------- output sink

// Counts when p == nullptr (length pass), writes otherwise (write pass): both passes run the same formatting code.
struct Sink {
    uint8_t *p;
    int64_t n;
    KC_HD void put(uint8_t c) {
        if (p) p[n] = c;
        ++n;
    }
    KC_HD void put(const uint8_t *s, uint32_t len) {
        if (p)
            for (uint32_t i = 0; i < len; ++i) p[n + i] = s[i];
        n += len;
    }
    KC_HD void lit(const char *s) {
        for (; *s; ++s) put((uint8_t)*s);
    }
    KC_HD void u_escape(uint32_t v) {  // \uxxxx, lower-case hex as json.dumps writes it
        put('\\');
        put('u');
        for (int k = 12; k >= 0; k -= 4) {
            const uint32_t d = (v >> k) & 15u;
            put((uint8_t)(d < 10 ? '0' + d : 'a' + d - 10));
        }
    }
    // json.dumps of one character of a string (ensure_ascii): `"` `\` and \n \r \t \b \f as two-character escapes, other
    // controls and DEL as \u00xx, printable ASCII as itself, the rest of the BMP (lone surrogates included) as \uxxxx, astral
    // code points as a surrogate pair.  The host path (kc_json.cpp) prints its strings through it as well.
    KC_HD void json_char(uint32_t cp) {
        if (cp == '"' || cp == '\\') {
            put('\\');
            put((uint8_t)cp);
        } else if (cp >= 0x20 && cp < 0x7F) {
            put((uint8_t)cp);
        } else if (cp == '\n' || cp == '\r' || cp == '\t' || cp == 8 || cp == 12) {
            put('\\');
            put(cp == '\n' ? 'n' : (cp == '\r' ? 'r' : (cp == '\t' ? 't' : (cp == 8 ? 'b' : 'f'))));
        } else if (cp >= 0x10000) {
            u_escape(0xD800u + ((cp - 0x10000u) >> 10));
            u_escape(0xDC00u + ((cp - 0x10000u) & 0x3FFu));
        } else {
            u_escape(cp);
        }
    }
    // json.dumps of a string value (ensure_ascii), quotes included, from its raw span (token flags: TOK_ESCAPED, TOK_UNICODE).
    // ASCII spans: the two-character escapes are already what json.dumps prints, except "\/", which it prints as "/".  TOK_UNICODE
    // spans are decoded to code points and printed one by one (json_char).  The length pass counts exactly what the write pass
    // writes: it is this same code.
    KC_HD void json_string(const uint8_t *s, uint32_t len, uint8_t flags) {
        put('"');
        if (flags & TOK_UNICODE) {
            for (uint32_t i = 0; i < len;) json_char(decode_cp(s, len, i));
        } else if (!(flags & TOK_ESCAPED)) {
            put(s, len);
        } else {
            for (uint32_t i = 0; i < len; ++i) {
                if (s[i] == '\\' && s[i + 1] == '/') continue;  // a backslash is never the span's last byte
                put(s[i]);
                if (s[i] == '\\') put(s[++i]);
            }
        }
        put('"');
    }
};

// ---------------------------------------------------------------- float64 -> float.__repr__ (Ryu shortest digits)

namespace ryu {

KC_HD inline const uint64_t *pow5_inv(uint32_t i) {
#ifdef __CUDA_ARCH__
    return ::kc::ryu::kPow5InvSplitDev[i];
#else
    return ::kc::ryu::kPow5InvSplitHost[i];
#endif
}
KC_HD inline const uint64_t *pow5(uint32_t i) {
#ifdef __CUDA_ARCH__
    return ::kc::ryu::kPow5SplitDev[i];
#else
    return ::kc::ryu::kPow5SplitHost[i];
#endif
}

KC_HD inline uint32_t pow5bits(int32_t e) { return (uint32_t)(((uint32_t)e * 1217359u) >> 19) + 1u; }  // ceil(log2(5^e)), 0 <= e <= 3528
KC_HD inline uint32_t log10_pow2(int32_t e) { return ((uint32_t)e * 78913u) >> 18; }                  // floor(log10(2^e)), 0 <= e <= 1650
KC_HD inline uint32_t log10_pow5(int32_t e) { return ((uint32_t)e * 732923u) >> 20; }                 // floor(log10(5^e)), 0 <= e <= 2620

KC_HD inline uint32_t pow5_factor(uint64_t v) {
    uint32_t c = 0;
    while (v && v % 5 == 0) {
        v /= 5;
        ++c;
    }
    return c;
}
KC_HD inline bool multiple_of_pow5(uint64_t v, uint32_t p) { return pow5_factor(v) >= p; }
KC_HD inline bool multiple_of_pow2(uint64_t v, uint32_t p) { return (v & ((1ull << p) - 1)) == 0; }

KC_HD inline uint64_t mul_shift(uint64_t m, const uint64_t *mul, int32_t j) {  // (m * mul) >> j, j >= 64
    const u128 b0 = (u128)m * mul[0];
    const u128 b2 = (u128)m * mul[1];
    return (uint64_t)(((b0 >> 64) + b2) >> (j - 64));
}

// Shortest decimal (digits, exponent) that reads back as the finite, non-zero double with these fields.
KC_HD inline void shortest(uint64_t ieee_mant, uint32_t ieee_exp, uint64_t &digits, int32_t &exp10) {
    int32_t e2;
    uint64_t m2;
    if (ieee_exp == 0) {
        e2 = 1 - 1023 - 52 - 2;
        m2 = ieee_mant;
    } else {
        e2 = (int32_t)ieee_exp - 1023 - 52 - 2;
        m2 = (1ull << 52) | ieee_mant;
    }
    const bool accept = (m2 & 1) == 0;
    const uint64_t mv = 4 * m2;
    const uint32_t mm_shift = (ieee_mant != 0 || ieee_exp <= 1) ? 1u : 0u;
    uint64_t vr, vp, vm;
    int32_t e10;
    bool vm_tz = false, vr_tz = false;
    if (e2 >= 0) {
        const uint32_t q = log10_pow2(e2) - (e2 > 3 ? 1u : 0u);
        e10 = (int32_t)q;
        const int32_t k = ::kc::ryu::kPow5InvBitCount + (int32_t)pow5bits((int32_t)q) - 1;
        const int32_t i = -e2 + (int32_t)q + k;
        const uint64_t *mul = pow5_inv(q);
        vr = mul_shift(4 * m2, mul, i);
        vp = mul_shift(4 * m2 + 2, mul, i);
        vm = mul_shift(4 * m2 - 1 - mm_shift, mul, i);
        if (q <= 21) {
            const uint32_t mv_mod5 = (uint32_t)(mv % 5);
            if (mv_mod5 == 0) vr_tz = multiple_of_pow5(mv, q);
            else if (accept) vm_tz = multiple_of_pow5(mv - 1 - mm_shift, q);
            else vp -= multiple_of_pow5(mv + 2, q) ? 1u : 0u;
        }
    } else {
        const uint32_t q = log10_pow5(-e2) - (-e2 > 1 ? 1u : 0u);
        e10 = (int32_t)q + e2;
        const int32_t i = -e2 - (int32_t)q;
        const int32_t k = (int32_t)pow5bits(i) - ::kc::ryu::kPow5BitCount;
        const int32_t j = (int32_t)q - k;
        const uint64_t *mul = pow5((uint32_t)i);
        vr = mul_shift(4 * m2, mul, j);
        vp = mul_shift(4 * m2 + 2, mul, j);
        vm = mul_shift(4 * m2 - 1 - mm_shift, mul, j);
        if (q <= 1) {
            vr_tz = true;
            if (accept) vm_tz = mm_shift == 1;
            else --vp;
        } else if (q < 63) {
            vr_tz = multiple_of_pow2(mv, q);
        }
    }
    int32_t removed = 0;
    uint32_t last = 0;
    uint64_t out;
    if (vm_tz || vr_tz) {
        for (;;) {
            const uint64_t vp10 = vp / 10, vm10 = vm / 10;
            if (vp10 <= vm10) break;
            const uint32_t vm_mod = (uint32_t)(vm - 10 * vm10);
            const uint64_t vr10 = vr / 10;
            const uint32_t vr_mod = (uint32_t)(vr - 10 * vr10);
            vm_tz &= vm_mod == 0;
            vr_tz &= last == 0;
            last = vr_mod;
            vr = vr10;
            vp = vp10;
            vm = vm10;
            ++removed;
        }
        if (vm_tz) {
            for (;;) {
                const uint64_t vm10 = vm / 10;
                const uint32_t vm_mod = (uint32_t)(vm - 10 * vm10);
                if (vm_mod != 0) break;
                const uint64_t vp10 = vp / 10, vr10 = vr / 10;
                const uint32_t vr_mod = (uint32_t)(vr - 10 * vr10);
                vr_tz &= last == 0;
                last = vr_mod;
                vr = vr10;
                vp = vp10;
                vm = vm10;
                ++removed;
            }
        }
        if (vr_tz && last == 5 && vr % 2 == 0) last = 4;  // exactly half: round to even
        out = vr + (((vr == vm && (!accept || !vm_tz)) || last >= 5) ? 1u : 0u);
    } else {
        bool round_up = false;
        for (;;) {
            const uint64_t vp10 = vp / 10, vm10 = vm / 10;
            if (vp10 <= vm10) break;
            const uint64_t vr10 = vr / 10;
            const uint32_t vr_mod = (uint32_t)(vr - 10 * vr10);
            round_up = vr_mod >= 5;
            vr = vr10;
            vp = vp10;
            vm = vm10;
            ++removed;
        }
        out = vr + ((vr == vm || round_up) ? 1u : 0u);
    }
    digits = out;
    exp10 = e10 + removed;
}

}  // namespace ryu

// json.dumps(x) for a float: float.__repr__ (fixed notation for -4 <= exponent10 < 16, else d[.ddd]e+XX; always a fractional
// part), NaN / Infinity / -Infinity spelled the JSON way.
KC_HD inline void float_repr(double x, Sink &o) {
    const uint64_t bits = f64_bits(x);
    const bool neg = (bits >> 63) != 0;
    const uint32_t ieee_exp = (uint32_t)((bits >> 52) & 0x7FF);
    const uint64_t ieee_mant = bits & 0xFFFFFFFFFFFFFull;
    if (ieee_exp == 0x7FF) {
        if (ieee_mant) o.lit("NaN");
        else o.lit(neg ? "-Infinity" : "Infinity");
        return;
    }
    if (neg) o.put('-');
    if (ieee_exp == 0 && ieee_mant == 0) {
        o.lit("0.0");
        return;
    }
    uint64_t digits;
    int32_t exp10;
    ryu::shortest(ieee_mant, ieee_exp, digits, exp10);
    uint8_t buf[20];
    int nd = 0;
    while (digits) {
        buf[nd++] = (uint8_t)('0' + digits % 10);
        digits /= 10;
    }  // buf holds the digits least-significant first
    const int decpt = exp10 + nd;  // position of the decimal point relative to the first digit
    if (decpt > 16 || decpt < -3) {
        o.put(buf[nd - 1]);
        if (nd > 1) {
            o.put('.');
            for (int i = nd - 2; i >= 0; --i) o.put(buf[i]);
        }
        o.put('e');
        int e = decpt - 1;
        o.put(e < 0 ? '-' : '+');
        if (e < 0) e = -e;
        if (e >= 100) o.put((uint8_t)('0' + e / 100));
        o.put((uint8_t)('0' + (e / 10) % 10));
        o.put((uint8_t)('0' + e % 10));
    } else if (decpt <= 0) {
        o.lit("0.");
        for (int i = 0; i < -decpt; ++i) o.put('0');
        for (int i = nd - 1; i >= 0; --i) o.put(buf[i]);
    } else if (decpt >= nd) {
        for (int i = nd - 1; i >= 0; --i) o.put(buf[i]);
        for (int i = 0; i < decpt - nd; ++i) o.put('0');
        o.lit(".0");
    } else {
        for (int i = nd - 1; i >= 0; --i) {
            if (nd - 1 - i == decpt) o.put('.');
            o.put(buf[i]);
        }
    }
}

}  // namespace js
}  // namespace kc
