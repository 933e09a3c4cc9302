// kc_json.cpp — H1: native host columnariser / decoder (SURVEY.md §8f-1).
//
// kc_consolidate_json(): for every record, n candidate JSON texts in -> consensus JSON text + likelihoods JSON text out,
// with only the CUDA kernels in between.  It does, in C++ and multi-threaded, what the reference does per request in
// Python around the hot path:
//     _safe_parse_content            consolidation.py:25-38   (json.loads, or {"text": content})
//     recursive_list_alignments      consensus_utils.py:516-548 (dict part: every candidate gets every key, keys SORTED)
//     consensus_values dispatcher    consensus_utils.py:1376-1454 (scalar fields, nested objects, lists element-wise)
//     lists_alignment                consensus_utils.py:185-430 + majority_sorting.py (H2 below; records with list fields)
//     sanitize_value / `v or False`  consensus_utils.py:925-933, 956   -> local dictionary codes (int8 cells)
//     _format_consensus_content      consolidation.py:41-60   (json.dumps of the consensus; {"text": s} -> s)
//     similarity medoid              consensus_utils.py:1221-1237 for multi-word string fields (batched into one K4 launch)
// Records it cannot express (a key mixing objects with other types, string groups outside K4's contract, non-ASCII
// text, mixed-type bool groups) are NOT guessed at: they get status 1 and the Python path handles them.
//
// Text formats follow CPython exactly: float -> float.__repr__ (shortest round-trip digits, exponent form outside
// 1e-4 <= |x| < 1e16, always a fractional part), json.dumps separators ", " / ": " and ensure_ascii escaping.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <charconv>  // from_chars (kc_align.inl)
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/kllms_b200.h"
#include "kc_internal.h"    // kc_alignsim: element similarities of the alignment pre-pass (kc_alignsim.cuh)
#include "kc_jsoncore.cuh"  // to_double, float_repr: the device path's exact number conversions (host-callable)

namespace {

enum TokType : uint8_t { T_MISSING = 0, T_NULL, T_TRUE, T_FALSE, T_INT, T_FLOAT, T_STR, T_NESTED };

// A token is a VIEW into the candidate text (no copies): strings keep their raw inner span and an "has escapes" flag
// and are read character by character (each_char) where the value is needed; numbers keep their text span and the strtod value.
struct Tok {
    TokType type = T_MISSING;
    bool esc = false;
    const char *p = nullptr;
    uint32_t len = 0;
    double num = 0.0;  // T_INT / T_FLOAT (strtod: correctly rounded, like float(int) / float(text))
};

struct Item {
    std::string_view key;  // raw span; empty for a list element
    bool kesc = false;     // the key holds escapes (only aligned texts may: json.dumps escapes quotes, backslashes, controls)
    Tok tok;
};

// f(c) for each character of a string given by its span: with `esc` (a raw JSON span holding escapes) each escape is decoded
// by kc::js::decode_cp; every other byte is one character.  A span without escapes is the value itself, and it need not be
// JSON: the {"text": ...} wrapper is a decoded value, in which a backslash is a backslash.
template <typename F>
void each_char(const char *p, uint32_t len, bool esc, F f) {
    const uint8_t *s = (const uint8_t *)p;
    for (uint32_t i = 0; i < len;) {
        if (esc && s[i] == '\\') f(kc::js::decode_cp(s, len, i));
        else f((uint32_t)s[i++]);
    }
}

// the value of a string from its span, one byte per character (H1 declines \uXXXX escapes above 0x7F)
void str_value(const char *p, uint32_t len, bool esc, std::string &out) {
    out.clear();
    if (!esc) out.assign(p, len);
    else each_char(p, len, true, [&](uint32_t c) { out.push_back((char)c); });
}

struct Scanner {
    const char *p, *end;
    bool non_ascii = false;
    void ws() {
        while (p < end && kc::js::is_json_ws((uint8_t)*p)) ++p;
    }
    bool lit(const char *s, size_t n) {
        if ((size_t)(end - p) >= n && memcmp(p, s, n) == 0) {
            p += n;
            return true;
        }
        return false;
    }
    // at the opening quote: validates, reports the raw inner span
    bool string(const char *&sp, uint32_t &slen, bool &esc) {
        ++p;
        sp = p;
        esc = false;
        while (p < end) {
            const unsigned char c = (unsigned char)*p;
            if (c == '"') {
                slen = (uint32_t)(p - sp);
                ++p;
                return true;
            }
            if (c < 0x20) return false;  // json.loads(strict=True) rejects raw control characters
            if (c >= 0x80) non_ascii = true;
            if (c != '\\') {
                ++p;
                continue;
            }
            esc = true;
            if (++p >= end) return false;
            const char k = *p++;
            if (k == 'u') {
                uint32_t v;
                if (end - p < 4 || !kc::js::hex4((const uint8_t *)p, v)) return false;
                p += 4;
                if (v >= 0x80) non_ascii = true;  // parity for non-ASCII text is unpinned: hand the record to Python
            } else if (!(k == '"' || k == '\\' || k == '/' || k == 'b' || k == 'f' || k == 'n' || k == 'r' || k == 't')) {
                return false;
            }
        }
        return false;
    }
    // at '{' or '[': validate the nested value exactly as json.loads would (a malformed inner value makes the WHOLE candidate
    // text invalid JSON, which the caller then treats as free text, consolidation.py:25-38) and skip it
    bool skip_nested(int depth = 0) {
        if (depth > 200) return false;
        const char open = *p++;
        const char close = open == '{' ? '}' : ']';
        ws();
        if (p < end && *p == close) {
            ++p;
            return true;
        }
        for (;;) {
            ws();
            if (open == '{') {
                if (p >= end || *p != '"') return false;
                const char *sp;
                uint32_t sl;
                bool esc;
                if (!string(sp, sl, esc)) return false;
                ws();
                if (p >= end || *p != ':') return false;
                ++p;
            }
            Tok inner;
            if (!value(inner, depth + 1)) return false;
            ws();
            if (p < end && *p == ',') {
                ++p;
                continue;
            }
            if (p < end && *p == close) {
                ++p;
                return true;
            }
            return false;
        }
    }
    bool number(Tok &t) {
        const char *s = p;
        if (p < end && *p == '-') ++p;
        if (p >= end) return false;
        if (*p == '0') {
            ++p;
        } else if (*p >= '1' && *p <= '9') {
            while (p < end && *p >= '0' && *p <= '9') ++p;
        } else {
            return false;
        }
        bool is_float = false;
        if (p < end && *p == '.') {
            ++p;
            if (p >= end || *p < '0' || *p > '9') return false;
            while (p < end && *p >= '0' && *p <= '9') ++p;
            is_float = true;
        }
        if (p < end && (*p == 'e' || *p == 'E')) {
            const char *q = p + 1;
            if (q < end && (*q == '+' || *q == '-')) ++q;
            if (q < end && *q >= '0' && *q <= '9') {
                while (q < end && *q >= '0' && *q <= '9') ++q;
                p = q;
                is_float = true;
            }
        }
        t.p = s;
        t.len = (uint32_t)(p - s);
        t.type = is_float ? T_FLOAT : T_INT;
        if (kc::js::to_double((const uint8_t *)s, t.len, t.num)) {
            // the exact integer-arithmetic conversion of the device path (kc_jsoncore.cuh: <= 19 significant digits, checked against
            // CPython on 280 k texts), several times faster than strtod; texts beyond its range fall through to strtod
        } else if (t.len < 40) {  // strtod needs a terminated buffer
            char buf[40];
            memcpy(buf, s, t.len);
            buf[t.len] = 0;
            t.num = strtod(buf, nullptr);
        } else {
            t.num = strtod(std::string(s, t.len).c_str(), nullptr);
        }
        return true;
    }
    bool value(Tok &t, int depth = 0) {
        ws();
        if (p >= end) return false;
        const char c = *p;
        if (c == '"') {
            t.type = T_STR;
            return string(t.p, t.len, t.esc);
        }
        if (c == '{' || c == '[') {
            t.type = T_NESTED;
            t.p = p;
            const bool ok = skip_nested(depth);
            t.len = (uint32_t)(p - t.p);
            return ok;
        }
        if (c == 't' && lit("true", 4)) { t.type = T_TRUE; return true; }
        if (c == 'f' && lit("false", 5)) { t.type = T_FALSE; return true; }
        if (c == 'n' && lit("null", 4)) { t.type = T_NULL; return true; }
        if (c == 'N' && lit("NaN", 3)) { t.type = T_FLOAT; t.num = NAN; return true; }
        if (c == 'I' && lit("Infinity", 8)) { t.type = T_FLOAT; t.num = INFINITY; return true; }
        if (c == '-' && lit("-Infinity", 9)) { t.type = T_FLOAT; t.num = -INFINITY; return true; }
        return number(t);
    }
};

// json.loads(text) one level deep: an object's (key, value) items or, with `lists`, a list's elements (empty keys).  `object`
// tells whether it was an object; anything else that json.loads would ACCEPT (top-level list, number, ...) has no members.
// A parse failure means the reference wraps the text (consolidation.py:37-38).  `odd` is set for escaped keys.
bool parse_members(const char *s, size_t len, bool lists, std::vector<Item> &out, bool &object, bool &non_ascii, bool &odd) {
    Scanner sc{s, s + len};
    out.clear();
    sc.ws();
    if (sc.p >= sc.end) return false;
    const char open = *sc.p;
    object = open == '{';
    if (!object && (open != '[' || !lists)) {
        Tok t;
        const bool ok = sc.value(t);
        sc.ws();
        non_ascii = sc.non_ascii;
        return ok && sc.p == sc.end;
    }
    const char close = object ? '}' : ']';
    ++sc.p;
    sc.ws();
    if (sc.p < sc.end && *sc.p == close) {
        ++sc.p;
    } else {
        for (;;) {
            Item it;
            if (object) {
                sc.ws();
                if (sc.p >= sc.end || *sc.p != '"') return false;
                const char *kp;
                uint32_t kl;
                if (!sc.string(kp, kl, it.kesc)) return false;
                odd |= it.kesc;
                sc.ws();
                if (sc.p >= sc.end || *sc.p != ':') return false;
                ++sc.p;
                it.key = std::string_view(kp, kl);
            }
            if (!sc.value(it.tok)) return false;
            out.push_back(it);
            sc.ws();
            if (sc.p < sc.end && *sc.p == ',') {
                ++sc.p;
                continue;
            }
            if (sc.p < sc.end && *sc.p == close) {
                ++sc.p;
                break;
            }
            return false;
        }
    }
    sc.ws();
    non_ascii = sc.non_ascii;
    return sc.p == sc.end;
}

// a.key < b.key in byte order of the decoded keys (code-point order for ASCII, consensus_utils.py:521-522)
bool key_less(const Item &a, const Item &b) {
    if (!a.kesc && !b.kesc) return a.key < b.key;
    thread_local std::string x, y;
    str_value(a.key.data(), (uint32_t)a.key.size(), a.kesc, x);
    str_value(b.key.data(), (uint32_t)b.key.size(), b.kesc, y);
    return x < y;
}

// "reasoning___" in key or "source___" in key (cu:1292), on the decoded key
bool special_key(const Item &k) {
    thread_local std::string decoded;
    std::string_view key = k.key;
    if (k.kesc) {
        str_value(k.key.data(), (uint32_t)k.key.size(), true, decoded);
        key = decoded;
    }
    return key.find("reasoning___") != std::string_view::npos || key.find("source___") != std::string_view::npos;
}

// ---------------------------------------------------------------- CPython text formats

// json.dumps(x) for a float: float.__repr__, NaN / Infinity / -Infinity spelled the JSON way (kc::js::float_repr)
void put_float(double x, std::string &out) {
    uint8_t buf[32];  // the longest repr is 24 characters
    kc::js::Sink o{buf, 0};
    kc::js::float_repr(x, o);
    out.append((const char *)buf, (size_t)o.n);
}

// json.dumps(str) with ensure_ascii=True of a string given by its span (each_char), quotes included: every character through
// the device path's kc::js::Sink::json_char
void json_string(const char *p, uint32_t len, bool esc, std::string &out) {
    const size_t k = out.size();
    out.resize(k + 6 * (size_t)len + 2);  // json_char prints at most six bytes per byte of the span (a surrogate pair: twelve for twelve)
    kc::js::Sink o{(uint8_t *)out.data() + k, 0};
    o.put('"');
    each_char(p, len, esc, [&](uint32_t c) { o.json_char(c); });
    o.put('"');
    out.resize(k + (size_t)o.n);
}
void json_string(std::string_view s, std::string &out) { json_string(s.data(), (uint32_t)s.size(), false, out); }  // a decoded string

// str(int) of a JSON integer token: the digits as written (JSON forbids leading zeros), except "-0" -> "0"
void int_text(const Tok &t, std::string &out) {
    if (t.len == 2 && t.p[0] == '-' && t.p[1] == '0') out += "0";
    else out.append(t.p, t.len);
}

// str(v) of a bool or number token as Python prints it (the vote classes sanitise it like a string)
void py_str(const Tok &t, std::string &out) {
    switch (t.type) {
        case T_TRUE: out += "True"; break;
        case T_FALSE: out += "False"; break;
        case T_INT: int_text(t, out); break;
        case T_FLOAT:  // str(float): repr, but non-finite values spelled nan / inf / -inf
            if (std::isnan(t.num)) out += "nan";
            else if (std::isinf(t.num)) out += t.num < 0 ? "-inf" : "inf";
            else put_float(t.num, out);
            break;
        default: break;
    }
}

// sanitize_value(s) (consensus_utils.py:925-933; == normalize_string, :660-673, on ASCII) of a string given by its span
// (each_char): the characters kc::js::is_alnum_lower keeps, lower-cased.  Returns len(s).
uint32_t sanitized(const char *p, uint32_t len, bool esc, std::string &out) {
    out.resize(len);  // at most one character per byte: written in place, trimmed once (no per-character capacity checks)
    char *o = out.data();
    size_t k = 0;
    uint32_t chars = 0;
    each_char(p, len, esc, [&](uint32_t c) {
        uint8_t b = (uint8_t)c;
        const bool keep = c < 0x80 && kc::js::is_alnum_lower(b);
        o[k] = (char)b;
        k += keep ? 1 : 0;
        ++chars;
    });
    out.resize(k);
    return chars;
}

void json_value(const Tok &t, std::string &out) {
    switch (t.type) {
        case T_TRUE: out += "true"; break;
        case T_FALSE: out += "false"; break;
        case T_INT: int_text(t, out); break;
        case T_FLOAT: put_float(t.num, out); break;
        case T_STR: json_string(t.p, t.len, t.esc, out); break;
        default: out += "null"; break;
    }
}

// ---------------------------------------------------------------- per-record plan

enum GroupKind : uint8_t { G_ALLNULL = 0, G_VOTE_STR, G_VOTE_BOOL, G_NUMERIC, G_MEDOID };

struct Group {
    GroupKind kind;
    int64_t row = -1;       // row in the vote / numeric cell matrix, or the medoid group index
    uint32_t m_first = 0;   // G_MEDOID: first string of the group in Record::mlen, and how many (the non-None cells)
    uint32_t m_count = 0;
};

// Shape of the consensus object: a dict node lists its children (sorted keys), a leaf points at its group.
struct Node {
    std::string_view key;      // raw span of the key (Item::key / kesc)
    bool kesc = false;
    int32_t group = -1;        // >= 0: leaf
    bool is_list = false;      // a list node: children are its columns, in order (no keys)
    std::vector<int32_t> kids; // dict / list: indices into Record::nodes
};

struct Record {
    uint8_t status = 0;        // 0 native, 1 needs the Python path, 2 (while planning) has list fields: align, then plan again
    std::vector<Node> nodes;   // nodes[0] is the root dict
    std::vector<Group> groups;
    std::vector<Tok> cells;    // groups.size() * n tokens, group-major (T_MISSING / T_NULL count as None)
    std::string mchars;        // normalize_string() of the cells of the medoid groups, back to back
    std::vector<int32_t> mlen; // their lengths
    std::vector<std::string> aligned;  // records with lists: the aligned candidate texts the cells and keys point into
};

const double kF64None = [] { const uint64_t b = KC_F64_NONE_BITS; double d; memcpy(&d, &b, 8); return d; }();

// Scalar field: which kernel decides it (cu:1405-1411 vote, cu:1443-1453 numeric / medoid).  False: Python path.
bool plan_leaf(Record &rec, Group &g, const Tok *cells, int n) {
    const Tok *first = nullptr;
    for (int c = 0; c < n && !first; ++c)
        if (cells[c].type > T_NULL) first = &cells[c];
    if (!first) {
        g.kind = G_ALLNULL;
    } else if (first->type == T_NESTED) {
        rec.status = 1;
        return false;
    } else if (first->type == T_STR || first->type == T_TRUE || first->type == T_FALSE) {
        bool multi_word = false, all_str = true;
        int live = 0;
        for (int c = 0; c < n; ++c) {
            const Tok &t = cells[c];
            if (t.type <= T_NULL) continue;
            ++live;
            if (t.type == T_NESTED) {  // str(dict) is almost never enum-like: leave it to Python
                rec.status = 1;
                return false;
            }
            all_str &= t.type == T_STR;
            if (t.type == T_STR) {  // numbers and bools print as one word
                int words = 0;      // len(s.split())
                bool in = false;
                each_char(t.p, t.len, t.esc, [&](uint32_t ch) {
                    const bool sp = kc::js::is_py_space(ch);
                    words += (!sp && !in) ? 1 : 0;
                    in = !sp;
                });
                multi_word |= words >= 3;
            }
        }
        if (multi_word) {
            // Not enum-like (cu:1405): the similarity medoid of consensus_as_primitive (cu:1221-1237).  K4 takes it when
            // every pair is a Levenshtein pair inside its contract (same rule as columnar.Plan._medoid_on_device under
            // the default string_similarity_method "embeddings"); anything else goes to the Python path.
            if (!all_str) {
                rec.status = 1;
                return false;
            }
            g.kind = G_MEDOID;
            g.m_first = (uint32_t)rec.mlen.size();
            g.m_count = (uint32_t)live;
            if (live >= 2) {
                int long_raw = 0, long_norm = 0;
                thread_local std::string norm;
                for (int c = 0; c < n; ++c) {
                    const Tok &t = cells[c];
                    if (t.type != T_STR) continue;
                    long_raw += sanitized(t.p, t.len, t.esc, norm) > 50;  // len(s) > 50
                    long_norm += norm.size() > 64;
                    if (norm.size() > 2000 || long_raw > 1 || long_norm > 1) {
                        rec.status = 1;
                        return false;
                    }
                    rec.mchars += norm;
                    rec.mlen.push_back((int32_t)norm.size());
                }
            }
            return true;
        }
        if (first->type == T_STR) {
            g.kind = G_VOTE_STR;
        } else {
            for (int c = 0; c < n; ++c)  // `v or False` on non-bool values compares Python objects: Python path
                if (cells[c].type > T_FALSE) {
                    rec.status = 1;
                    return false;
                }
            g.kind = G_VOTE_BOOL;
        }
    } else {
        g.kind = G_NUMERIC;
    }
    return true;
}

// Depth bounds: on the texts as given, objects nested at most 15 below the root (16 levels of objects, whose fields sit one
// level deeper); on aligned texts, any value at most 48 below it (49 levels of the value tree, fields included).
constexpr int kMaxObjectDepth = 15, kMaxValueDepth = 48;

// One node of the alignment pre-pass + dispatcher (cu:516-548, cu:550-613, then cu:1414-1426): `items[c]` is candidate c's
// members here (an object's items sorted by key, or a list's elements), or nullptr where it holds None — the pre-pass turns
// None into an object or list of Nones, so parent_valid_frac stays 1.  The children (keys in sorted order, or a list's
// columns in order) whose values are all objects or all lists recurse; scalar fields go to plan_leaf; a mix of objects,
// lists and scalars sends the record to the Python path.  On the texts as given a list sets status 2: the record goes
// through the alignment pre-pass and is planned again on its `aligned` texts, where a list node holds lists of one width.
struct LevelScratch {  // per recursion depth, reused across records (no allocation in the steady state)
    std::vector<const Item *> keys;
    std::vector<size_t> cursor;
    std::vector<Tok> cells;
    std::vector<std::vector<Item>> child_items;
    std::vector<const std::vector<Item> *> child;
};

void plan_node(Record &rec, int32_t node, const std::vector<Item> *const *items, int n, int depth, bool aligned) {
    thread_local std::vector<LevelScratch> levels(kMaxValueDepth + 1);  // sized once: references stay valid through the recursion
    LevelScratch &L = levels[(size_t)depth];
    const bool list = rec.nodes[(size_t)node].is_list;
    std::vector<const Item *> &keys = L.keys;
    keys.clear();
    size_t width = 0;
    for (int c = 0; c < n; ++c)
        if (items[c]) {
            if (list) {
                width = items[c]->size();
                break;
            }
            for (auto &it : *items[c]) keys.push_back(&it);
        }
    if (!list) {
        std::sort(keys.begin(), keys.end(), [](const Item *a, const Item *b) { return key_less(*a, *b); });
        keys.erase(std::unique(keys.begin(), keys.end(), [](const Item *a, const Item *b) { return a->key == b->key; }), keys.end());
        width = keys.size();
    }
    std::vector<size_t> &cursor = L.cursor;
    cursor.assign((size_t)n, 0);
    std::vector<Tok> &cells = L.cells;
    cells.resize((size_t)n);
    for (size_t ki = 0; ki < width; ++ki) {
        const std::string_view key = list ? std::string_view() : keys[ki]->key;
        for (int c = 0; c < n; ++c) {  // merge: both sides are sorted by key; of duplicates the last one wins
            cells[(size_t)c] = Tok();
            if (!items[c]) continue;
            const auto &its = *items[c];
            size_t &k = cursor[(size_t)c];
            if (list) cells[(size_t)c] = its[ki].tok;
            else
                while (k < its.size() && its[k].key == key) cells[(size_t)c] = its[k++].tok;
        }
        if (!list && special_key(*keys[ki])) continue;
        const Tok *first = nullptr;
        for (int c = 0; c < n && !first; ++c)
            if (cells[(size_t)c].type > T_NULL) first = &cells[(size_t)c];
        const bool nested = first && first->type == T_NESTED;
        if (nested && *first->p == '[' && !aligned) {
            rec.status = 2;
            return;
        }
        if ((nested || aligned) && depth + 1 > (aligned ? kMaxValueDepth : kMaxObjectDepth)) {
            rec.status = 1;
            return;
        }
        const int32_t kid = (int32_t)rec.nodes.size();
        rec.nodes.emplace_back();
        rec.nodes[(size_t)kid].key = key;
        rec.nodes[(size_t)kid].kesc = !list && keys[ki]->kesc;
        rec.nodes[(size_t)node].kids.push_back(kid);
        if (nested) {
            auto &child_items = L.child_items;
            if ((int)child_items.size() < n) child_items.resize((size_t)n);
            auto &child = L.child;
            child.assign((size_t)n, nullptr);
            const size_t fc = (size_t)(first - cells.data());
            for (size_t c = fc; c < (size_t)n; ++c) {
                const Tok &t = cells[c];
                if (t.type <= T_NULL) continue;
                if (t.type != T_NESTED || *t.p != *first->p) {  // not all of one type: the pre-pass leaves the values alone (cu:507-512)
                    rec.status = 1;
                    return;
                }
                bool object = false, non_ascii = false, odd = false;
                if (!parse_members(t.p, t.len, true, child_items[c], object, non_ascii, odd) || non_ascii || (odd && !aligned) ||
                    (!object && child_items[c].size() != child_items[fc].size())) {
                    rec.status = 1;
                    return;
                }
                std::stable_sort(child_items[c].begin(), child_items[c].end(), key_less);
                child[c] = &child_items[c];
            }
            rec.nodes[(size_t)kid].is_list = *first->p == '[';
            plan_node(rec, kid, child.data(), n, depth + 1, aligned);
            if (rec.status) return;
            continue;
        }
        const size_t base = rec.cells.size();
        rec.cells.insert(rec.cells.end(), cells.begin(), cells.end());
        Group g;
        if (!plan_leaf(rec, g, &rec.cells[base], n)) return;
        rec.nodes[(size_t)kid].group = (int32_t)rec.groups.size();
        rec.groups.push_back(g);
    }
}

// Plans a record from its n candidate texts, or (`aligned`) from the texts the alignment pre-pass made of them.
void plan_record(const char *const *texts, const int64_t *lens, int n, Record &rec, bool aligned) {
    thread_local std::vector<std::vector<Item>> cands;
    if ((int)cands.size() < n) cands.resize((size_t)n);
    static const char kTextKey[] = "text";
    rec.status = 0;
    for (int c = 0; c < n; ++c) {
        const char *s = texts[c];
        const size_t len = lens ? (size_t)lens[c] : strlen(s);
        if (len == 0) {  // `if choice.message.content:` drops empty contents, changing n (consolidation.py:92): Python path
            rec.status = 1;
            return;
        }
        bool object = false, non_ascii = false, odd = false;
        std::vector<Item> &items = cands[(size_t)c];
        const bool ok = parse_members(s, len, false, items, object, non_ascii, odd);
        if (!ok || !non_ascii)  // a failed parse may have stopped early: look at every byte
            for (size_t i = 0; i < len && !non_ascii; ++i)
                if ((unsigned char)s[i] >= 0x80) non_ascii = true;
        if (non_ascii || (odd && !aligned) || (ok && !object)) {
            rec.status = 1;
            return;
        }
        if (!ok) {  // {"text": content}: the whole text is the (already unescaped) value
            items.clear();
            Item it;
            it.key = std::string_view(kTextKey, 4);
            it.tok.type = T_STR;
            it.tok.p = s;
            it.tok.len = (uint32_t)len;
            items.push_back(it);
        }
        // sort by key; of duplicates the LAST one in the text wins (dict construction)
        std::stable_sort(items.begin(), items.end(), key_less);
    }
    rec.groups.clear();
    rec.cells.clear();
    rec.mchars.clear();
    rec.mlen.clear();
    rec.nodes.clear();
    rec.nodes.emplace_back();
    thread_local std::vector<const std::vector<Item> *> top;
    top.assign((size_t)n, nullptr);
    for (int c = 0; c < n; ++c) top[(size_t)c] = &cands[(size_t)c];
    plan_node(rec, 0, top.data(), n, 0, aligned);
}

void encode_vote(GroupKind kind, const Tok *toks, int n, int8_t *cells) {
    thread_local std::vector<std::string> seen;
    thread_local std::string tmp, san;
    size_t n_seen = 0;
    for (int c = 0; c < n; ++c) {
        const Tok &t = toks[c];
        if (kind == G_VOTE_BOOL) {
            cells[c] = (t.type == T_TRUE) ? 1 : 0;  // None and False -> False (cu:956)
            continue;
        }
        if (t.type <= T_NULL) {
            cells[c] = KC_CODE_NONE;
            continue;
        }
        if (t.type == T_STR) {
            sanitized(t.p, t.len, t.esc, san);
        } else {
            tmp.clear();
            py_str(t, tmp);
            sanitized(tmp.data(), (uint32_t)tmp.size(), false, san);
        }
        size_t k = 0;
        while (k < n_seen && seen[k] != san) ++k;
        if (k == n_seen) {
            if (seen.size() <= n_seen) seen.emplace_back();
            seen[n_seen++] = san;
        }
        cells[c] = (int8_t)k;
    }
}

void encode_numeric(const Tok *toks, int n, double *cells) {
    for (int c = 0; c < n; ++c) {
        const Tok &t = toks[c];
        if (t.type <= T_NULL) cells[c] = kF64None;
        else if (t.type == T_INT || t.type == T_FLOAT) cells[c] = t.num;  // non-finite values are dropped by the kernel
        else cells[c] = NAN;                                               // bool / str / nested: counted, never clustered
    }
}

struct EmitCtx {
    const Record &rec;
    int n;
    const uint32_t *vmeta;
    const double *nvalue;
    const uint32_t *nmeta;
    const int32_t *midx;
    const double *mavg;
};

// value and confidence of one leaf group (the epilogue of cu:971-982, cu:1085-1086, cu:1116, cu:1177-1219, cu:1233-1237)
void emit_leaf(const EmitCtx &cx, size_t gi, std::string &content, std::string &lik) {
    const Record &rec = cx.rec;
    const int n = cx.n;
    const uint32_t *vmeta = cx.vmeta, *nmeta = cx.nmeta;
    const double *nvalue = cx.nvalue, *mavg = cx.mavg;
    const int32_t *midx = cx.midx;
    const Group &g = rec.groups[gi];
    const Tok *cells = &rec.cells[gi * (size_t)n];
        double conf = 0.0;
        Tok value;  // T_MISSING == None
        if (g.kind == G_VOTE_STR || g.kind == G_VOTE_BOOL) {
            const uint32_t m = vmeta[g.row];
            const uint32_t idx = KC_META_IDX(m);
            if (g.kind == G_VOTE_BOOL) {
                value.type = (cells[idx].type == T_TRUE) ? T_TRUE : T_FALSE;  // the processed key (cu:958)
            } else {
                value = cells[idx];  // first original whose sanitised form wins (cu:971)
            }
            // always the HAS_VALUE arm: a string group has a non-None cell, and a bool group turns None into False
            conf = kc::confidence(m, false, 1.0);
        } else if (g.kind == G_NUMERIC) {
            const uint32_t m = nmeta[g.row];
            const uint32_t flags = KC_META_FLAGS(m);
            if (flags & KC_FLAG_HAS_VALUE) {
                if (flags & KC_FLAG_SINGLE) {
                    value = cells[KC_META_IDX(m)];
                } else {
                    value.type = T_FLOAT;
                    value.num = nvalue[g.row];
                }
            }
            conf = kc::confidence(m, true, 1.0);
        } else if (g.kind == G_MEDOID) {
            int want = g.m_count >= 2 ? midx[g.row] : 0;
            for (int c = 0; c < n; ++c) {
                if (cells[c].type <= T_NULL) continue;
                if (want-- == 0) {
                    value = cells[c];
                    break;
                }
            }
            conf = kc::medoid_confidence(g.m_count, n, g.m_count >= 2 ? mavg[g.row] : 0.0);
        }  // G_ALLNULL: None, 0.0 (cu:1401-1402)
        json_value(value, content);
        put_float(conf, lik);
}

void emit_node(const EmitCtx &cx, int32_t ni, std::string &content, std::string &lik) {
    const Node &node = cx.rec.nodes[(size_t)ni];
    if (node.group >= 0) {
        emit_leaf(cx, (size_t)node.group, content, lik);
        return;
    }
    content += node.is_list ? "[" : "{";
    lik += node.is_list ? "[" : "{";
    bool first = true;
    for (int32_t kid : node.kids) {
        if (!first) {
            content += ", ";
            lik += ", ";
        }
        first = false;
        if (!node.is_list) {
            const Node &k = cx.rec.nodes[(size_t)kid];
            json_string(k.key.data(), (uint32_t)k.key.size(), k.kesc, content);
            json_string(k.key.data(), (uint32_t)k.key.size(), k.kesc, lik);
            content += ": ";
            lik += ": ";
        }
        emit_node(cx, kid, content, lik);
    }
    content += node.is_list ? "]" : "}";
    lik += node.is_list ? "]" : "}";
}

void emit_record(const Record &rec, int n, const uint32_t *vmeta, const double *nvalue, const uint32_t *nmeta, const int32_t *midx,
                 const double *mavg, std::string &content, std::string &lik) {
    const EmitCtx cx{rec, n, vmeta, nvalue, nmeta, midx, mavg};
    content.clear();
    lik.clear();
    emit_node(cx, 0, content, lik);
    // {"text": s} -> s (consolidation.py:55-57): a single top-level string field called "text"
    const Node &root = rec.nodes[0];
    if (root.kids.size() == 1) {
        const Node &only = rec.nodes[(size_t)root.kids[0]];
        if (only.group >= 0 && only.key == "text") {
            const Group &g = rec.groups[(size_t)only.group];
            const Tok *cells = &rec.cells[(size_t)only.group * (size_t)n];
            const Tok *picked = nullptr;
            if (g.kind == G_VOTE_STR) {
                picked = &cells[KC_META_IDX(vmeta[g.row])];
            } else if (g.kind == G_MEDOID) {
                int want = g.m_count >= 2 ? midx[g.row] : 0;
                for (int c = 0; c < n && !picked; ++c)
                    if (cells[c].type > T_NULL && want-- == 0) picked = &cells[c];
            }
            if (picked && picked->type == T_STR) {
                content.clear();
                str_value(picked->p, picked->len, picked->esc, content);
            }
        }
    }
}

char *dup_string(const std::string &s) {
    char *p = (char *)malloc(s.size() + 1);
    if (p) memcpy(p, s.c_str(), s.size() + 1);
    return p;
}

template <typename F>
void parallel_for(int64_t n, int threads, F fn) {
    std::atomic<int64_t> next{0};
    const int64_t grain = 256;
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t)
        pool.emplace_back([&] {
            for (;;) {
                const int64_t b = next.fetch_add(grain);
                if (b >= n) return;
                const int64_t e = std::min(n, b + grain);
                for (int64_t i = b; i < e; ++i) fn(i);
            }
        });
    for (auto &th : pool) th.join();
}


#include "kc_align.inl"  // H2: value tree, similarities, assignment, lists_alignment, recursive_list_alignments

// A record with list fields, planned again on the n texts the alignment pre-pass made of its candidates (status: the
// pre-pass's; non-zero sends the record to the Python path).  The record keeps the texts: its cells and keys point into them.
void plan_aligned(Record &rec, int status, std::vector<std::string> &aligned, int n) {
    if (status) {
        rec.status = 1;
        return;
    }
    rec.aligned = std::move(aligned);
    thread_local std::vector<const char *> texts;
    thread_local std::vector<int64_t> lens;
    texts.resize((size_t)n);
    lens.resize((size_t)n);
    for (int c = 0; c < n; ++c) {
        texts[(size_t)c] = rec.aligned[(size_t)c].data();
        lens[(size_t)c] = (int64_t)rec.aligned[(size_t)c].size();
    }
    plan_record(texts.data(), lens.data(), n, rec, true);
}

// ---------------------------------------------------------------- a batch of records: plan, encode, emit

struct Batch {
    int n = 0;
    std::vector<Record> recs;
    int64_t gv = 0, gx = 0, gm = 0;       // vote / numeric / medoid groups of the records with status 0
    std::vector<uint8_t> m_chars;         // medoid groups of the whole batch in CSR form for ONE K4 launch
    std::vector<int32_t> m_str_off{0}, m_grp_off{0};
    int32_t m_max_group = 2;
};

int default_threads() { return (int)std::min(32u, std::max(1u, std::thread::hardware_concurrency())); }  // parsing saturates memory / malloc beyond ~32

// Records with list fields are aligned (H2, under the ConsensusSettings default min_support_ratio 0.51, cu:41) and planned again
// on their aligned texts.  sim_device >= 0: the element similarities of their list nodes come from one kc_alignsim pass on that
// device (the records are aligned after it); < 0: each similarity is computed on the host when the alignment asks for it.
int plan_batch(Batch &b, const char *const *texts, const int64_t *lens, int64_t n_records, int n, int threads, int sim_device) {
    b.n = n;
    b.recs.assign((size_t)n_records, Record());
    parallel_for(n_records, threads, [&](int64_t r) { plan_record(texts + r * n, lens ? lens + r * n : nullptr, n, b.recs[(size_t)r], false); });
    std::vector<int64_t> idx;  // the records with list fields; a candidate that is not JSON is aligned as {"text": content}
    for (int64_t r = 0; r < n_records; ++r)
        if (b.recs[(size_t)r].status == 2) idx.push_back(r);
    const int64_t m = (int64_t)idx.size();
    if (sim_device >= 0 && m) {
        std::vector<const char *> sub_texts((size_t)(m * n));
        std::vector<int64_t> sub_lens(lens ? (size_t)(m * n) : 0);
        for (int64_t i = 0; i < m; ++i)
            for (int c = 0; c < n; ++c) {
                sub_texts[(size_t)(i * n + c)] = texts[idx[(size_t)i] * n + c];
                if (lens) sub_lens[(size_t)(i * n + c)] = lens[idx[(size_t)i] * n + c];
            }
        const int rc = align_batch(sub_texts.data(), lens ? sub_lens.data() : nullptr, m, n, 0.51, true, sim_device, threads,
                                   nullptr, [&](int64_t i, int status, std::vector<std::string> &aligned) { plan_aligned(b.recs[(size_t)idx[(size_t)i]], status, aligned, n); });
        if (rc) return rc;
    } else if (m) {
        parallel_for(m, threads, [&](int64_t i) {
            const int64_t r = idx[(size_t)i];
            std::vector<std::string> aligned;
            const int status = align_record(texts + r * n, lens ? lens + r * n : nullptr, n, 0.51, true, aligned);
            plan_aligned(b.recs[(size_t)r], status, aligned, n);
        });
    }
    for (auto &rec : b.recs) {
        if (rec.status) continue;
        for (auto &g : rec.groups) {
            if (g.kind == G_VOTE_STR || g.kind == G_VOTE_BOOL) g.row = b.gv++;
            else if (g.kind == G_NUMERIC) g.row = b.gx++;
            else if (g.kind == G_MEDOID && g.m_count >= 2) {
                g.row = b.gm++;
                for (uint32_t k = 0; k < g.m_count; ++k) b.m_str_off.push_back(b.m_str_off.back() + rec.mlen[g.m_first + k]);
                b.m_grp_off.push_back(b.m_grp_off.back() + (int32_t)g.m_count);
                b.m_max_group = std::max(b.m_max_group, (int32_t)g.m_count);
            }
        }
        if (!rec.mchars.empty()) b.m_chars.insert(b.m_chars.end(), rec.mchars.begin(), rec.mchars.end());
    }
    return KC_OK;
}

void encode_batch(const Batch &b, int8_t *codes, double *vals, int threads) {
    const int n = b.n;
    parallel_for((int64_t)b.recs.size(), threads, [&](int64_t r) {
        const Record &rec = b.recs[(size_t)r];
        if (rec.status) return;
        for (size_t gi = 0; gi < rec.groups.size(); ++gi) {
            const Group &g = rec.groups[gi];
            const Tok *toks = &rec.cells[gi * (size_t)n];
            if (g.kind == G_VOTE_STR || g.kind == G_VOTE_BOOL) encode_vote(g.kind, toks, n, codes + g.row * n);
            else if (g.kind == G_NUMERIC) encode_numeric(toks, n, vals + g.row * n);
        }
    });
}

void emit_batch(const Batch &b, const uint32_t *vmeta, const double *nvalue, const uint32_t *nmeta, const int32_t *midx, const double *mavg,
                int threads, char **out_content, char **out_likelihoods, uint8_t *out_status) {
    parallel_for((int64_t)b.recs.size(), threads, [&](int64_t r) {
        const Record &rec = b.recs[(size_t)r];
        out_status[r] = rec.status;
        out_content[r] = nullptr;
        out_likelihoods[r] = nullptr;
        if (rec.status) return;
        std::string content, lik;
        emit_record(rec, b.n, vmeta, nvalue, nmeta, midx, mavg, content, lik);
        out_content[r] = dup_string(content);
        out_likelihoods[r] = dup_string(lik);
    });
}

}  // namespace

extern "C" {

int kc_consolidate_json(const char *const *texts, const int64_t *lens, int64_t n_records, int32_t n, double rel_eps,
                        double abs_eps, int device, int32_t threads, char **out_content, char **out_likelihoods,
                        uint8_t *out_status) {
    if (n < 2 || n > KC_MAX_CANDIDATES || n_records < 0 || !texts || !out_content || !out_likelihoods || !out_status)
        return KC_EINVAL;
    if (threads <= 0) threads = default_threads();
    const bool timing = getenv("KC_JSON_TIMING") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = now();
    Batch batch;
    if (const int rc = plan_batch(batch, texts, lens, n_records, n, threads, device)) return rc;
    const auto t1 = now();
    const int64_t gv = batch.gv, gx = batch.gx, gm = batch.gm;
    std::vector<int32_t> m_idx((size_t)gm);
    std::vector<double> m_avg((size_t)gm);
    // page-locked staging buffers are expensive to create: keep them (grow-only) across calls, never destroyed
    static std::mutex pool_mu;
    static kc::GrowBuf<kc::Mem::Pinned> *const pool = new kc::GrowBuf<kc::Mem::Pinned>[6];
    std::lock_guard<std::mutex> pool_lock(pool_mu);  // also serialises callers (one staging pool per process)
    auto pinned = [&](int slot, size_t bytes) { return bytes && pool[slot].reserve(bytes) == KC_OK ? pool[slot].p : nullptr; };
    int8_t *h_codes = (int8_t *)pinned(0, (size_t)gv * n);
    double *h_vals = (double *)pinned(1, (size_t)gx * n * 8);
    int32_t *h_win = (int32_t *)pinned(2, (size_t)gv * 4);
    uint32_t *h_vmeta = (uint32_t *)pinned(3, (size_t)gv * 4);
    double *h_value = (double *)pinned(4, (size_t)gx * 8);
    uint32_t *h_nmeta = (uint32_t *)pinned(5, (size_t)gx * 4);
    const auto t2 = now();
    auto t3 = t2, t4 = t2;
    int rc = KC_OK;
    if ((gv && (!h_codes || !h_win || !h_vmeta)) || (gx && (!h_vals || !h_value || !h_nmeta))) rc = KC_ENOMEM;
    if (!rc) {
        encode_batch(batch, h_codes, h_vals, threads);
        t3 = now();
        // one "field" per group: the two halves are independent calls of the host-buffer entry
        if (gv) rc = kc_consensus_host_i8(h_codes, 1, nullptr, nullptr, 0, gv, n, rel_eps, abs_eps, h_win, h_vmeta, nullptr, nullptr, device, nullptr);
        if (!rc && gx) rc = kc_consensus_host_i8(nullptr, 0, nullptr, h_vals, 1, gx, n, rel_eps, abs_eps, nullptr, nullptr, h_value, h_nmeta, device, nullptr);
        if (!rc && gm)
            rc = kc_medoid_str_host(batch.m_chars.data(), (int64_t)batch.m_chars.size(), batch.m_str_off.data(), batch.m_grp_off.data(), gm,
                                    batch.m_max_group, m_idx.data(), m_avg.data(), device);
    }
    t4 = now();
    if (!rc) emit_batch(batch, h_vmeta, h_value, h_nmeta, m_idx.data(), m_avg.data(), threads, out_content, out_likelihoods, out_status);
    const auto t5 = now();
    if (timing)
        fprintf(stderr, "kc_consolidate_json: parse+plan %.1f ms, rows+alloc %.1f ms, encode %.1f ms, gpu %.1f ms, emit %.1f ms (%d threads)\n",
                ms(t0, t1), ms(t1, t2), ms(t2, t3), ms(t3, t4), ms(t4, t5), threads);
    return rc;
}

// The same in two phases, for callers that run K1 / K2 / K4 themselves (their own streams, another device, a test that puts
// a checker in their place): kc_json_plan parses, plans and encodes a batch into host arrays the handle owns; the caller
// computes the result columns for them; kc_json_emit turns those into the consensus texts.  The candidate texts must stay
// alive until kc_json_emit returns (cells are views into them).
struct kc_json_batch {
    Batch batch;
    std::vector<int8_t> codes;
    std::vector<double> vals;
    int threads;
};

int kc_json_plan(const char *const *texts, const int64_t *lens, int64_t n_records, int32_t n, int32_t threads, kc_json_batch **out) {
    if (n < 2 || n > KC_MAX_CANDIDATES || n_records < 0 || !texts || !out) return KC_EINVAL;
    if (threads <= 0) threads = default_threads();
    kc_json_batch *h = new (std::nothrow) kc_json_batch;
    if (!h) return KC_ENOMEM;
    h->threads = threads;
    if (const int rc = plan_batch(h->batch, texts, lens, n_records, n, threads, -1)) {
        delete h;
        return rc;
    }
    h->codes.resize((size_t)h->batch.gv * n);
    h->vals.resize((size_t)h->batch.gx * n);
    encode_batch(h->batch, h->codes.data(), h->vals.data(), threads);
    *out = h;
    return KC_OK;
}

int kc_json_inputs(const kc_json_batch *h, const int8_t **vote_cells, int64_t *n_vote_groups, const double **num_cells,
                   int64_t *n_num_groups, const uint8_t **medoid_chars, const int32_t **medoid_str_off, const int32_t **medoid_grp_off,
                   int64_t *n_medoid_groups, int32_t *max_medoid_group) {
    if (!h) return KC_EINVAL;
    if (vote_cells) *vote_cells = h->codes.data();
    if (n_vote_groups) *n_vote_groups = h->batch.gv;
    if (num_cells) *num_cells = h->vals.data();
    if (n_num_groups) *n_num_groups = h->batch.gx;
    if (medoid_chars) *medoid_chars = h->batch.m_chars.data();
    if (medoid_str_off) *medoid_str_off = h->batch.m_str_off.data();
    if (medoid_grp_off) *medoid_grp_off = h->batch.m_grp_off.data();
    if (n_medoid_groups) *n_medoid_groups = h->batch.gm;
    if (max_medoid_group) *max_medoid_group = h->batch.m_max_group;
    return KC_OK;
}

int kc_json_emit(kc_json_batch *h, const uint32_t *vote_meta, const double *num_value, const uint32_t *num_meta, const int32_t *medoid_idx,
                 const double *medoid_avg, char **out_content, char **out_likelihoods, uint8_t *out_status) {
    if (!h || !out_content || !out_likelihoods || !out_status) return KC_EINVAL;
    if ((h->batch.gv && !vote_meta) || (h->batch.gx && (!num_value || !num_meta)) || (h->batch.gm && (!medoid_idx || !medoid_avg))) return KC_EINVAL;
    emit_batch(h->batch, vote_meta, num_value, num_meta, medoid_idx, medoid_avg, h->threads, out_content, out_likelihoods, out_status);
    return KC_OK;
}

void kc_json_free(kc_json_batch *h) { delete h; }

// H2: recursive_list_alignments(values, "embeddings", embed, client, min_support_ratio)[0] for ONE record of n candidate
// values given as JSON texts (null = None): out_texts[c] = json.dumps of candidate c's aligned value (free with
// kc_free_strings).  Returns 0; 1 if the record needs the Python path (a pair of strings both longer than 50 characters
// would be compared through embeddings, cu:813; non-ASCII text); negative for invalid JSON.
int kc_align_json(const char *const *texts, const int64_t *lens, int32_t n, double min_support_ratio, char **out_texts) {
    if (!texts || !out_texts || n < 1) return KC_EINVAL;
    for (int32_t c = 0; c < n; ++c) out_texts[c] = nullptr;
    std::vector<std::string> aligned;
    if (const int status = align_record(texts, lens, n, min_support_ratio, false, aligned)) return status;
    for (int32_t c = 0; c < n; ++c) out_texts[c] = dup_string(aligned[(size_t)c]);
    return 0;
}

// kc_align_json for a batch of records (n candidate texts each, record-major), with the element similarities of their list
// nodes computed in one kc_alignsim pass on `device` (< 0: the same phase on the host) before the records are aligned.
int kc_align_json_batch(const char *const *texts, const int64_t *lens, int64_t n_records, int32_t n, double min_support_ratio, int device,
                        int32_t threads, char **out_texts, int32_t *out_status, int64_t *out_counts) {
    if (!texts || !out_texts || !out_status || n < 1 || n_records < 0) return kc_fail(KC_EINVAL, "kc_align_json_batch: bad arguments");
    if (threads <= 0) threads = default_threads();
    for (int64_t i = 0; i < n_records * n; ++i) out_texts[i] = nullptr;
    const int rc = align_batch(texts, lens, n_records, n, min_support_ratio, false, device, threads, out_counts,
                               [&](int64_t r, int status, const std::vector<std::string> &aligned) {
                                   out_status[r] = status;
                                   if (!status)
                                       for (int32_t c = 0; c < n; ++c) out_texts[r * n + c] = dup_string(aligned[(size_t)c]);
                               });
    if (rc) kc_free_strings(out_texts, n_records * n);
    return rc;
}

// The similarity phase of kc_align_json_batch instantiated on the host for one node whose T elements are given as JSON
// texts: out[i * T + j] as kc_alignsim computes it (NaN where it leaves the pair to the host).  Test hook.  Returns the
// number of pairs i < j it decided, KC_EINVAL on invalid / non-ASCII JSON or T outside [2, 512].
int kc_debug_alignsim(const char *const *texts, int32_t T, double *out) { return kc_debug_alignsim_nodes(texts, &T, 1, 1, -1, out); }

// The same for n_nodes list nodes in one kc_alignsim pass: node g holds the next node_len[g] texts, its T x T matrix follows
// the previous node's in out.  device >= 0 launches the kernel; device < 0 runs the phase on the host with `lanes` lanes.
int kc_debug_alignsim_nodes(const char *const *texts, const int32_t *node_len, int32_t n_nodes, int32_t lanes, int device, double *out) {
    if (!texts || !node_len || !out || n_nodes < 1 || lanes < 1) return KC_EINVAL;
    AlignCtx cx;
    int64_t k = 0;
    for (int32_t g = 0; g < n_nodes; ++g) {
        const int32_t T = node_len[g];
        if (T < 2 || T > 512) return KC_EINVAL;
        const int32_t list = cx.tr.add(A_LIST);
        for (int32_t i = 0; i < T; ++i, ++k) {
            Scanner sc{texts[k], texts[k] + strlen(texts[k])};
            int32_t id;
            if (!aparse(sc, cx.tr, id, 0) || sc.non_ascii) return KC_EINVAL;
            sc.ws();
            if (sc.p != sc.end) return KC_EINVAL;
            cx.tr.v[(size_t)list].items.push_back(id);
        }
        sim_add_node(cx, std::vector<int32_t>{list}, cx.sims);
    }
    int64_t pairs = 0;
    const SimTable &t = cx.sims;
    const int rc = kc_alignsim(t.nodes.data(), (int64_t)t.nodes.size(), t.vals.data(), (int64_t)t.vals.size(),
                               reinterpret_cast<const uint8_t *>(t.chars.data()), (int64_t)t.chars.size(), out, t.out_len, device, lanes, &pairs);
    if (rc) return rc;
    return pairs > INT32_MAX ? kc_fail(KC_EINVAL, "kc_debug_alignsim_nodes: more than 2^31 pairs") : (int)pairs;
}

// generic_similarity (consensus_utils.py:892-917, default string method) of two JSON values; test hook of the native alignment.
// Returns 0 and *out, 1 if a pair of long strings would need embeddings, negative on invalid JSON.
int kc_debug_similarity_json(const char *a, const char *b, double *out) {
    AlignCtx cx;
    int32_t ia, ib;
    Scanner sa{a, a + strlen(a)}, sb{b, b + strlen(b)};
    if (!aparse(sa, cx.tr, ia, 0) || !aparse(sb, cx.tr, ib, 0) || sa.non_ascii || sb.non_ascii) return KC_EINVAL;
    sa.ws();
    sb.ws();
    if (sa.p != sa.end || sb.p != sb.end) return KC_EINVAL;
    // pointers into the vector: no insertion happens below
    *out = generic_similarity(cx, &cx.tr.v[(size_t)ia], &cx.tr.v[(size_t)ib]);
    return cx.decline ? 1 : 0;
}

// scipy.optimize.linear_sum_assignment(cost) restated (test hook): pairs sorted by row; returns their count or -1.
int kc_debug_lsap(int32_t nr, int32_t nc, const double *cost, int32_t *row_ind, int32_t *col_ind) {
    std::vector<int> rows, cols;
    if (!lsap(nr, nc, cost, rows, cols)) return -1;
    for (size_t k = 0; k < rows.size(); ++k) {
        row_ind[k] = rows[k];
        col_ind[k] = cols[k];
    }
    return (int)rows.size();
}

// Unit-cost edit distance of two byte strings (what python-Levenshtein's `distance` returns for the ASCII strings
// normalize_string() produces, consensus_utils.py:745-761).  Host helper for the similarity medoid / list alignment.
int32_t kc_levenshtein(const char *a, int32_t alen, const char *b, int32_t blen) {
    if (alen < 0 || blen < 0 || (!a && alen) || (!b && blen)) return -1;
    if (alen < blen) {
        std::swap(a, b);
        std::swap(alen, blen);
    }
    if (blen == 0) return alen;
    thread_local std::vector<int32_t> row;
    row.resize((size_t)blen + 1);
    for (int32_t j = 0; j <= blen; ++j) row[(size_t)j] = j;
    for (int32_t i = 1; i <= alen; ++i) {
        int32_t diag = row[0];
        row[0] = i;
        const char ca = a[i - 1];
        for (int32_t j = 1; j <= blen; ++j) {
            const int32_t up = row[(size_t)j];
            const int32_t v = std::min(std::min(up + 1, row[(size_t)j - 1] + 1), diag + (ca != b[j - 1] ? 1 : 0));
            diag = up;
            row[(size_t)j] = v;
        }
    }
    return row[(size_t)blen];
}

void kc_free_strings(char **arr, int64_t count) {
    if (!arr) return;
    for (int64_t i = 0; i < count; ++i) {
        free(arr[i]);
        arr[i] = nullptr;
    }
}

}  // extern "C"
