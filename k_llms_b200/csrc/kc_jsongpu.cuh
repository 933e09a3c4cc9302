// kc_jsongpu.cuh — H1g: the JSON-in / JSON-out path of the consolidator ON THE DEVICE.
//
// The reference's unit of work is n candidate JSON texts -> consensus JSON (+ likelihoods): json.loads per candidate
// (consolidation.py:25-38), the dict part of recursive_list_alignments (consensus_utils.py:516-548: every candidate gets
// every key, keys SORTED), the dispatcher (:1376-1454), sanitize_value (:925-933), the vote / numeric consensus (K1 / K2),
// and json.dumps of the result (consolidation.py:41-60).  Round 1 did everything around K1/K2 on host threads (H1,
// kc_json.cpp): 211 k records/s against 2 G records/s for the kernels.  Here the candidate texts are copied to the GPU as
// they are and the GPU does the whole chain; the host only moves bytes:
//
//   A0  count_kernel    one thread per record scans candidate 0 -> number of fields F_r        (then an exclusive scan: slots)
//   A1  plan_kernel     a TEAM of lanes per record (team size = n rounded up to a power of two, <= 32):
//         parse   lane c scans candidate c, one 16-byte token (key span, value span, kind) per field
//         type    lane j (one per token): same shape in every candidate (same keys, nested objects open / close at the same
//                 positions), duplicate / special keys, rank of the key among its siblings in sorted order, which kernel
//                 decides the field (plan_leaf of kc_json.cpp)
//         order   nested records: the token's position in output order (depth-first, keys sorted at every level)
//         slots   the team leader numbers the record's vote / numeric groups and reserves rows in the batch's cell matrices
//         encode  lane j: sanitised-equality classes -> int8 local codes (K1 cells), exact decimal -> float64 (K2 cells)
//   U1-U3 only under KC_JSON_KEY_UNION and when A1 found records whose candidates differ in SHAPE (keys in another order,
//         missing or extra keys, None or nothing where another candidate holds a sub-object): the key-union round, a team per
//         such record (without the flag A1 declines them)
//     U1  union_count_kernel   lane c counts candidate c's tokens; the leader reserves scratch        (read-back: scratch size)
//     U2  union_build_kernel   lane c scans candidate c into scratch; the leader builds the union tree (one node per key path,
//                              duplicate keys and object-against-value declined) and reserves its rows  (read-back: union rows)
//     U3  union_plan_kernel    lane c writes column c of the [union rows x n] table (synthetic K_NULL / K_OPEN..K_CLOSE where
//                              candidate c lacks the key or holds None), then type / order / slots / encode run on it as in A1
//   list round          only under KC_JSON_LISTS and when A1 marked records D_LIST (some candidate holds a list): after the
//                       call's chunks the host aligns them (H2, kc_align_json_batch) and the chunks run again over the aligned
//                       texts with list nodes on (Chunk::lists = 2: K_LOPEN / K_LCLOSE tokens, keyless TOK_ELEM elements ranked
//                       by their index), every stage from A0 to C1 unchanged otherwise (kc_jsongpu.cu, list_round)
//   A2  medoid_kernel   only when the chunk has multi-word string fields (three exclusive scans of the per-record counts first):
//                       lane j writes its field's normalised strings and their offsets in K4's CSR form
//   K1  kc_vote_i8, K2  kc_numeric_f64, K4  kc_medoid_str on the cell matrices / string groups — the kernels of the columnar path
//   C0  len_kernel      lane j formats its field's value and confidence (float.__repr__ by Ryu) to learn the lengths; the
//                       leader turns them into piece offsets and record lengths          (then two exclusive scans: offsets)
//   C1  write_kernel    lane j writes `"key": value` / `"key": confidence` at its offset of the two output blobs
//
// A record the device path does not model exactly (\u escapes, DEL and non-ASCII without KC_JSON_UNICODE, or with it in vote fields,
// escapes, DEL and non-ASCII in keys, lists without KC_JSON_LISTS, empty objects, an object in one
// candidate against a value in another, candidates of different shapes without KC_JSON_KEY_UNION, multi-word strings outside
// K4's contract, numbers outside the exact-conversion range, ...) gets a non-zero status and is
// consolidated by the host path (kc_consolidate_json) instead: the device path never guesses.
//
// The phases are plain __host__ __device__ functions of (chunk, record, lane, team size) that communicate through global
// arrays only — no warp intrinsics.  Each kernel's schedule of phases is one step function over a team type (the steps at the
// end of this file): the kernels run it with a team of lanes, the host twin (kc_debug_jsongpu_*) with a loop over the lanes,
// so the CPU tests run the SAME phases in the SAME order as the kernels.
#pragma once

#include "kc_jsoncore.cuh"

namespace kc {
namespace js {

constexpr int32_t kMaxFields = 1024;  // per record; the key ranking is quadratic in it

// status of a record between A1 and the union round (U1-U3): its candidates differ in shape.  Internal: the union round turns
// it into 0 or a D_* code before anything reads the statuses back.
constexpr uint8_t D_UNION = 0xFF;
// status of a record after the first round under KC_JSON_LISTS: some candidate holds a list and none is declined for another
// reason.  The list round aligns it on the host and consolidates the aligned texts in a round of its own.
constexpr uint8_t D_LIST = 0xFE;

// A node of a record's key-union tree (union round): one key path.  Indices are relative to the record's scratch region;
// node 0 is the top-level object.
struct UNode {
    uint32_t kstart;           // key span of the first candidate that has the key
    uint16_t klen;
    uint8_t depth;
    uint8_t obj;               // an object in some candidate
    uint8_t scalar;            // a non-null scalar in some candidate
    int32_t parent, child, last, next;  // tree links, -1 = none; members in order of first appearance
    int32_t lastc;             // the last candidate that has the key (a second hit from the same one is a duplicate key)
    uint32_t row, close;       // its row in the union table; an object's K_CLOSE row (the root: the node count in `row`)
};

// field descriptor word: kind:4 | last of its siblings in output order:1 | rank among its siblings:11 | group index within the
// record:16.  The rank of a member is its key's position in sorted order, of a list element its index.
KC_HD inline uint32_t fdesc_pack(uint32_t kind, uint32_t last, uint32_t rank, uint32_t gidx) { return kind | (last << 4) | (rank << 5) | (gidx << 16); }
KC_HD inline uint32_t fdesc_kind(uint32_t d) { return d & 15u; }
KC_HD inline uint32_t fdesc_last(uint32_t d) { return (d >> 4) & 1u; }
KC_HD inline uint32_t fdesc_rank(uint32_t d) { return (d >> 5) & 0x7FFu; }
KC_HD inline uint32_t fdesc_gidx(uint32_t d) { return d >> 16; }

struct Chunk {
    const uint8_t *text;  // the chunk's candidate texts (device copy), text[0] is byte off[0] of the caller's blob
    const int64_t *off;   // [R*n + 1] byte offsets of the candidate texts in the caller's blob (record-major)
    int32_t R, n;
    uint32_t *fcount;   // [R]   A0: tokens of candidate 0 (0 when it does not scan)
    uint8_t *nest;      // [R]   A0: 1 when candidate 0 holds a nested object
    uint32_t *gpos;     // [slots] nested records only: the token's position in OUTPUT order (sorted keys at every level)
    uint32_t *slot;     // [R+1] exclusive scan of fcount: the record's first field slot
    uint8_t *status;    // [R]   0 = on the device path, else D_*
    Tok *toks;          // [slots * n] token of (field slot, candidate)
    uint32_t *fdesc;    // [slots]
    uint32_t *vbase, *xbase;        // [R] first vote / numeric group of the record
    unsigned long long *counters;   // [0] vote groups, [1] numeric groups, [2] medoid groups of the chunk
    int8_t *vcells;     // [vote groups][n]   K1 cells
    double *xcells;     // [numeric groups][n] K2 cells
    // medoid fields (multi-word strings): per record the groups of >= 2 strings, their strings and normalised characters;
    // after the exclusive scans (in place, entry R = the totals) the record's first group / string / character
    uint32_t *mcount, *scount, *ccount;  // [R+1]
    uint8_t *mchars;                     // K4 input: normalised strings back to back
    int32_t *mstr_off, *mgrp_off;        //           [strings + 1], [groups + 1]
    const int32_t *midx;                 // K4 results: medoid's index within its group,
    const double *mavg;                  //             its mean similarity
    int32_t *vrec;           // [vote groups] or NULL: the (chunk-local) record of each vote group, for K3b over ragged records
    const float *vweight;    // [vote groups] or NULL: K3b's weights — the vote leaves are likelihood-weighted (DESIGN.md §5)
    const uint32_t *vmeta;   // K1 (or K3b) result words
    const double *xvalue;    // K2 values
    const uint32_t *xmeta;   // K2 result words
    // KC_JSON_NUMERIC_MEDOID (the reference's async dispatcher): numeric fields are similarity medoids, decided by K5 in K2's place
    bool xmedoid;
    const int32_t *xbest;    // K5 results: the medoid's position among the group's non-None cells,
    const double *xavg;      //             its mean similarity
    uint32_t *piece_c, *piece_l;  // [slots] by (slot + rank): piece length, then (after the leader's pass) piece offset
    int64_t *len_c, *len_l;       // [R+1] record lengths -> (exclusive scan, in place) record offsets in the output blobs
    uint8_t *out_c, *out_l;       // output blobs: consensus texts, likelihoods texts
    // the union round: records whose candidates differ in shape (key order, missing keys, null sub-objects), rebuilt as
    // [union rows x n] tables behind the first round's slots; counters [3] records, [4] scratch entries, [5] union rows
    uint8_t *pend;      // [R]   A1: a candidate's token count or a row's key / depth / structure differs from candidate 0's
    int32_t *plist;     // [R]   the records sent to the union round (chunk-local)
    uint32_t *ucand;    // [P*n] U1: candidate c's token count -> its first entry in the record's scratch region
    uint32_t *ubase;    // [P]   the record's scratch region
    uint32_t *usize;    // [P]   its size
    Tok *utok;          // [scratch] the candidates' tokens, back to back
    UNode *unode;       // [scratch] the union tree
    int32_t *umap;      // [scratch] token -> node (-1: a K_CLOSE)
    uint32_t uslot;     // the first round's slot total: union rows are numbered from here
    bool key_union;     // KC_JSON_KEY_UNION: such records go to the union round; without it A1 declines them as the reason says
    // KC_JSON_LISTS.  lists: 0 = a list declines the record (D_NESTED); 1 = first round: a record with a list in some candidate
    // is marked for the list round (lst), D_LIST unless a candidate declines it for another reason; 2 = aligned round: the
    // texts are the alignment pre-pass's output, list nodes are consolidated.  Records [aligned0, R) are in the aligned round
    // whatever `lists` says (the host twin runs both rounds in one chunk; the device runs them as chunks of their own).
    uint8_t *lst;       // [R]   A1: some candidate holds a list (first round)
    uint8_t lists;
    int32_t aligned0;
    // KC_JSON_UNICODE: string values may hold non-ASCII text and \uXXXX escapes (TOK_UNICODE tokens).  Similarity medoids take
    // them (normalize_string drops every non-ASCII code point); a vote field with one declines (its classes need unidecode).
    bool unicode;
};

KC_HD inline uint8_t load_status(const Chunk &ch, int32_t r) { return *(volatile const uint8_t *)(ch.status + r); }
KC_HD inline void decline(const Chunk &ch, int32_t r, int32_t why) { *(volatile uint8_t *)(ch.status + r) = (uint8_t)why; }
KC_HD inline uint32_t list_mode(const Chunk &ch, int32_t r) { return r >= ch.aligned0 ? 2u : ch.lists; }
// the candidates differ in shape (`why`: how A1 sees it): with KC_JSON_KEY_UNION the union round decides the record
// (D_KEYS_DIFFER keeps the later phases off it until then), else it is declined.  Aligned texts have one shape by construction:
// the union round never takes them.
KC_HD inline void differ(const Chunk &ch, int32_t r, int32_t why) {
    if (ch.key_union && list_mode(ch, r) != 2) {
        *(volatile uint8_t *)(ch.pend + r) = 1;
        why = D_KEYS_DIFFER;
    }
    decline(ch, r, why);
}

// ---------------------------------------------------------------- A0

KC_HD inline void count_record(const Chunk &ch, int32_t r) {
    const int64_t b = ch.off[(int64_t)r * ch.n], e = ch.off[(int64_t)r * ch.n + 1];
    int32_t f = -D_TOO_LONG;
    bool nested = false;
    if (e - b < ((int64_t)1 << 31))
        f = scan_object(ch.text + (b - ch.off[0]), (uint32_t)(e - b), 0, nullptr, 0, kMaxFields, &nested, list_mode(ch, r) != 0, nullptr,
                        ch.unicode);
    ch.fcount[r] = f > 0 ? (uint32_t)f : 0u;
    ch.nest[r] = nested ? 1 : 0;
    ch.pend[r] = 0;
    if (ch.lst) ch.lst[r] = 0;
    ch.status[r] = f > 0 ? (uint8_t)D_OK : (uint8_t)(-f);
}

// ---------------------------------------------------------------- A1

KC_HD inline void parse_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    const uint32_t mode = list_mode(ch, r);
    // first round under KC_JSON_LISTS: every lane scans its candidates whatever the other lanes found (a list in any candidate
    // sends the record to the list round, on every schedule of the lanes), unless candidate 0 did not scan (fcount 0)
    if (mode == 1 ? ch.fcount[r] == 0 : load_status(ch, r) != 0) return;
    const int32_t F = (int32_t)ch.fcount[r];
    const int64_t base0 = ch.off[0];
    for (int32_t c = lane; c < ch.n; c += team) {
        const int64_t b = ch.off[(int64_t)r * ch.n + c], e = ch.off[(int64_t)r * ch.n + c + 1];
        int32_t f = -D_TOO_LONG;
        bool listed = false;
        if (e - b < ((int64_t)1 << 31) && (b - base0) + (e - b) < ((int64_t)1 << 32)) {
            const uint8_t *s = ch.text + (b - base0);
            f = scan_object(s, (uint32_t)(e - b), (uint32_t)(b - base0), ch.toks + (int64_t)ch.slot[r] * ch.n + c, ch.n, F, nullptr, mode != 0, &listed,
                            ch.unicode);
            // first round: whether a candidate longer than candidate 0 holds a list past the tokens it has room for (a text
            // without a '[' byte holds none: the key-union records of the first round skip the full scan)
            if (mode == 1 && f == -D_TOO_MANY_FIELDS && !listed && contains(s, (uint32_t)(e - b), "[", 1))
                scan_object(s, (uint32_t)(e - b), 0, nullptr, 0, kMaxFields, nullptr, true, &listed, ch.unicode);
        }
        if (mode == 1 && listed) {  // the list round's record: slots_phase settles its status
            *(volatile uint8_t *)(ch.lst + r) = 1;
            decline(ch, r, D_LIST);
        } else if (f == -D_TOO_MANY_FIELDS || (f >= 0 && f != F)) {
            differ(ch, r, D_KEYS_DIFFER);  // more or fewer tokens than candidate 0
        } else if (f < 0) {
            decline(ch, r, -f);
        }
    }
}

// First round, team leader, a record with a list in some candidate: the first candidate (in order) declined for a reason of
// its own gives the record's reason, else it goes to the list round.  (Lanes that scanned in parallel may have left any of
// their reasons in the status; this makes the outcome the same on every schedule.)
KC_HD inline void settle_listed(const Chunk &ch, int32_t r) {
    int32_t why = D_LIST;
    for (int32_t c = 0; c < ch.n && why == D_LIST; ++c) {
        int64_t b, len;
        const int64_t base0 = ch.off[0];
        b = ch.off[(int64_t)r * ch.n + c] - base0;
        len = ch.off[(int64_t)r * ch.n + c + 1] - base0 - b;
        int32_t f = -D_TOO_LONG;
        if (len < ((int64_t)1 << 31)) f = scan_object(ch.text + b, (uint32_t)len, 0, nullptr, 0, kMaxFields, nullptr, true, nullptr, ch.unicode);
        if (f < 0) why = -f;
    }
    decline(ch, r, why);
}

// The siblings of a token at depth d: the tokens of depth d (other than K_CLOSE) in [lo, hi), the widest range around it in which
// no token is shallower.  A flat record: every token.
KC_HD inline void sibling_range(const Tok *rt, int32_t n, int32_t F, int32_t j, uint32_t d, bool flat, int32_t &lo, int32_t &hi) {
    lo = 0;
    hi = F;
    if (flat) return;
    lo = j;
    while (lo > 0 && tok_depth(rt[(int64_t)(lo - 1) * n]) >= d) --lo;
    hi = j + 1;
    while (hi < F && tok_depth(rt[(int64_t)hi * n]) >= d) ++hi;
}

KC_HD inline void type_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    if (load_status(ch, r)) return;
    const int32_t F = (int32_t)ch.fcount[r], n = ch.n;
    const bool flat = ch.nest[r] == 0;
    const Tok *rt = ch.toks + (int64_t)ch.slot[r] * n;
    for (int32_t j = lane; j < F; j += team) {
        const Tok *row = rt + (int64_t)j * n;
        const uint32_t k0 = row[0].kind, d = tok_depth(row[0]);
        // the same SHAPE in every candidate: the same key at position j, nested objects (and lists: aligned texts, where every
        // list of a node has one width) open and close at the same positions (else, with KC_JSON_KEY_UNION, the union round
        // applies the pre-pass's key union / missing -> None / None -> dict of Nones, cu:516-548; it also tells an object
        // against a non-null value, D_NESTED, from a row that is only out of step)
        int32_t ref = j;  // the token whose key orders this one among its siblings: itself, or a closer's opener
        if (is_close(k0)) {
            for (int32_t c = 1; c < n; ++c)
                if (row[c].kind != k0 || tok_depth(row[c]) != d) {
                    differ(ch, r, D_KEYS_DIFFER);
                    return;
                }
            ref = j - 1;  // its opener: the nearest token to the left at the same depth (everything between them is deeper)
            while (ref > 0 && tok_depth(rt[(int64_t)ref * n]) != d) --ref;
        }
        const uint8_t *key = ch.text + rt[(int64_t)ref * n].kstart;
        const uint32_t klen = rt[(int64_t)ref * n].klen;
        const uint8_t elem = rt[(int64_t)ref * n].flags & TOK_ELEM;
        if (!is_close(k0)) {
            for (int32_t c = 1; c < n; ++c) {
                if ((row[c].kind == K_OPEN) != (k0 == K_OPEN) || (row[c].kind == K_LOPEN) != (k0 == K_LOPEN) || is_close(row[c].kind)) {
                    differ(ch, r, D_NESTED);  // an object or a list here, a scalar / None / the other there
                    return;
                }
                if (tok_depth(row[c]) != d || (row[c].flags & TOK_ELEM) != elem || row[c].klen != klen ||
                    key_compare(ch.text + row[c].kstart, klen, key, klen) != 0) {
                    differ(ch, r, D_KEYS_DIFFER);
                    return;
                }
            }
            if (!elem && (contains(key, klen, "reasoning___", 12) || contains(key, klen, "source___", 9) ||  // skipped by consensus_dict (cu:1287-1294)
                          (F == 1 && klen == 4 && key_compare(key, 4, (const uint8_t *)"text", 4) == 0))) {   // {"text": s} -> s (cons:55-57)
                decline(ch, r, D_SPECIAL_KEY);
                return;
            }
        }
        // position of the key among its siblings in sorted order (cu:521-522, at every level); duplicates: dict semantics, host
        // path.  A list element's position is its index.
        int32_t lo, hi;
        sibling_range(rt, n, F, ref, d, flat, lo, hi);
        uint32_t rank = 0, after = 0;
        for (int32_t i = lo; i < hi; ++i) {
            const Tok &o = rt[(int64_t)i * n];
            if (i == ref || (!flat && (tok_depth(o) != d || is_close(o.kind)))) continue;
            if (elem) {
                rank += i < ref ? 1u : 0u;
                after += i > ref ? 1u : 0u;
                continue;
            }
            const int cmp = key_compare(ch.text + o.kstart, o.klen, key, klen);
            if (cmp == 0) {
                decline(ch, r, D_DUP_KEY);
                return;
            }
            rank += cmp < 0 ? 1u : 0u;
            after += cmp > 0 ? 1u : 0u;
        }
        const uint32_t last = after == 0 ? 1u : 0u;
        if (is_open(k0) || is_close(k0)) {
            const uint32_t kind = k0 == K_OPEN ? F_OPEN : (k0 == K_CLOSE ? F_CLOSE : (k0 == K_LOPEN ? F_LOPEN : F_LCLOSE));
            ch.fdesc[ch.slot[r] + j] = fdesc_pack(kind, last, rank, 0);
            continue;
        }
        // which kernel decides the field (plan_leaf, kc_json.cpp; cu:1405-1411, :1443-1453)
        int32_t first = -1;
        for (int32_t c = 0; c < n && first < 0; ++c)
            if (row[c].kind != K_NULL) first = c;
        uint32_t kind;
        if (first < 0) {
            kind = F_ALLNULL;
        } else if (row[first].kind == K_STR) {
            kind = F_VOTE_STR;
            bool uni = false;
            for (int32_t c = 0; c < n; ++c) {
                if (row[c].kind == K_NULL) continue;
                if (row[c].kind != K_STR) {  // str(v) of numbers / bools inside a string field: host path
                    decline(ch, r, D_MIXED_TYPES);
                    return;
                }
                if (row[c].flags & TOK_MULTIWORD) kind = F_MEDOID;  // not enum-like (cu:1405): the similarity medoid (cu:1221-1237)
                uni |= (row[c].flags & TOK_UNICODE) != 0;
            }
            if (kind == F_VOTE_STR && uni) {  // sanitize_value folds non-ASCII text through unidecode (cu:931): host path
                decline(ch, r, D_ESCAPE_OR_NON_ASCII);
                return;
            }
            if (kind == F_MEDOID) {
                // K4 takes the group when every pair is a Levenshtein pair inside its contract (plan_leaf of kc_json.cpp, the
                // rule of columnar.Plan._medoid_on_device under the default similarity method): at most one string longer than
                // 50 characters (two would go to the embeddings service, cu:813), at most one normalised string longer than 64
                uint32_t live = 0, chars = 0, long_raw = 0, long_norm = 0;
                bool fits = true;
                for (int32_t c = 0; c < n; ++c) {
                    if (row[c].kind == K_NULL) continue;
                    const uint8_t *v = ch.text + row[c].vstart;
                    const uint32_t vl = row[c].vlen;
                    const bool u = (row[c].flags & TOK_UNICODE) != 0;
                    const uint32_t nl = u ? normalize_string(v, vl, nullptr) : sanitized_copy(v, vl, nullptr);
                    ++live;
                    chars += nl;
                    // len(str): code points
                    const uint32_t raw = u ? code_points(v, vl) : ((row[c].flags & TOK_ESCAPED) ? unescaped_length(v, vl) : vl);
                    long_raw += raw > 50u ? 1u : 0u;
                    long_norm += nl > 64u ? 1u : 0u;
                    fits &= nl <= 2000u;
                }
                if (live >= 2 && (!fits || long_raw > 1 || long_norm > 1)) {
                    decline(ch, r, D_MULTIWORD);
                    return;
                }
                ch.piece_c[ch.slot[r] + j] = live;   // scratch until C0: read by the leader in slots_phase
                ch.piece_l[ch.slot[r] + j] = chars;
            }
        } else if (row[first].kind == K_TRUE || row[first].kind == K_FALSE) {
            kind = F_VOTE_BOOL;
            for (int32_t c = 0; c < n; ++c)
                if (row[c].kind > K_FALSE) {  // a string may be multi-word, `v or False` of other objects: host path
                    decline(ch, r, D_MIXED_TYPES);
                    return;
                }
        } else {
            kind = F_NUMERIC;  // strings / bools among the cells are "present, not a number" (cu:1105-1114)
            if (ch.xmedoid)    // ... but the async medoid compares them by generic_similarity's own rules (0 and false are both falsy)
                for (int32_t c = 0; c < n; ++c)
                    if (row[c].kind == K_STR || row[c].kind == K_TRUE || row[c].kind == K_FALSE) {
                        decline(ch, r, D_MIXED_TYPES);
                        return;
                    }
        }
        ch.fdesc[ch.slot[r] + j] = fdesc_pack(kind, last, rank, 0);
    }
}

// Nested records only, after type_phase: the token's position in output order.  Output is a depth-first walk with the members
// of every object in key order, so a token comes after its parent's K_OPEN and after the whole subtrees of the siblings that
// sort before it; a K_CLOSE comes last in its object's subtree.
KC_HD inline void order_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    if (load_status(ch, r) || ch.nest[r] == 0) return;
    const int32_t F = (int32_t)ch.fcount[r], n = ch.n;
    const Tok *rt = ch.toks + (int64_t)ch.slot[r] * n;
    const uint32_t *fd = ch.fdesc + ch.slot[r];
    auto subtree = [&](int32_t i) -> uint32_t {  // tokens in the subtree of token i (itself included)
        if (!is_open(rt[(int64_t)i * n].kind)) return 1u;
        const uint32_t d = tok_depth(rt[(int64_t)i * n]);
        int32_t e = i + 1;
        while (tok_depth(rt[(int64_t)e * n]) != d) ++e;  // its K_CLOSE / K_LCLOSE
        return (uint32_t)(e - i + 1);
    };
    for (int32_t j = lane; j < F; j += team) {
        const bool closing = is_close(rt[(int64_t)j * n].kind);
        uint32_t d = tok_depth(rt[(int64_t)j * n]);
        int32_t cur = j;
        if (closing) {
            cur = j - 1;
            while (cur > 0 && tok_depth(rt[(int64_t)cur * n]) != d) --cur;
        }
        uint32_t pos = closing ? subtree(cur) - 1u : 0u;
        for (;;) {
            int32_t lo, hi;
            sibling_range(rt, n, F, cur, d, false, lo, hi);
            const uint32_t rank = fdesc_rank(fd[cur]);
            for (int32_t i = lo; i < hi; ++i) {
                const Tok &o = rt[(int64_t)i * n];
                if (i == cur || tok_depth(o) != d || is_close(o.kind)) continue;
                if (fdesc_rank(fd[i]) < rank) pos += subtree(i);
            }
            if (d == 0) break;
            pos += 1u;     // the parent's K_OPEN, the token just before the first sibling
            cur = lo - 1;
            --d;
        }
        ch.gpos[ch.slot[r] + j] = pos;
    }
}

KC_HD inline uint32_t out_pos(const Chunk &ch, int32_t r, int32_t j) {
    return ch.nest[r] ? ch.gpos[ch.slot[r] + j] : fdesc_rank(ch.fdesc[ch.slot[r] + j]);
}

// team leader only: number the groups, reserve rows of the cell matrices (chunk-wide counters).  First round: a record whose
// candidates differ in shape goes to the union round, whatever else A1 found (the union round scans and checks it afresh).
KC_HD inline void slots_phase(const Chunk &ch, int32_t r, bool first_round) {
    if (first_round && ch.lst && ch.lst[r]) {
        settle_listed(ch, r);
        return;
    }
    if (load_status(ch, r)) {
        if (first_round && ch.pend[r]) {
            decline(ch, r, D_UNION);
#ifdef __CUDA_ARCH__
            ch.plist[atomicAdd(ch.counters + 3, 1ull)] = r;
#else
            ch.plist[ch.counters[3]++] = r;
#endif
        }
        return;
    }
    const int32_t F = (int32_t)ch.fcount[r];
    uint32_t *fd = ch.fdesc + ch.slot[r];
    uint32_t nv = 0, nx = 0, nm = 0, ns = 0, nc = 0;
    for (int32_t j = 0; j < F; ++j) {
        const uint32_t d = fd[j], kind = fdesc_kind(d);
        uint32_t g = 0;
        if (kind == F_VOTE_STR || kind == F_VOTE_BOOL) {
            g = nv++;
        } else if (kind == F_NUMERIC) {
            g = nx++;
        } else if (kind == F_MEDOID) {
            uint32_t *pc = ch.piece_c + ch.slot[r] + j, *pl = ch.piece_l + ch.slot[r] + j;
            const uint32_t live = *pc, chars = *pl;
            if (live >= 2) {  // one string alone is its own consensus (cu:1085-1086): no group
                g = nm++;
                *pc = ns;     // the group's first string / character within the record, for medoid_phase
                *pl = nc;
                ns += live;
                nc += chars;
            }
        }
        fd[j] = d | (g << 16);
    }
    ch.mcount[r] = nm;
    ch.scount[r] = ns;
    ch.ccount[r] = nc;
#ifdef __CUDA_ARCH__
    ch.vbase[r] = (uint32_t)atomicAdd(ch.counters + 0, (unsigned long long)nv);
    ch.xbase[r] = (uint32_t)atomicAdd(ch.counters + 1, (unsigned long long)nx);
    if (nm) atomicAdd(ch.counters + 2, (unsigned long long)nm);
#else
    ch.vbase[r] = (uint32_t)ch.counters[0];
    ch.counters[0] += nv;
    ch.xbase[r] = (uint32_t)ch.counters[1];
    ch.counters[1] += nx;
    ch.counters[2] += nm;
#endif
    if (ch.vrec)
        for (uint32_t k = 0; k < nv; ++k) ch.vrec[ch.vbase[r] + k] = r;
}

// A2, after the exclusive scans of mcount / scount / ccount: lane j writes its medoid group in K4's CSR form.  Group, string
// and character ranges follow RECORD order (scans, not atomics), so the three offset arrays are monotonic as CSR needs.  A
// record that was declined after slots_phase (a number out of range) still owns its ranges and fills them: K4 reads every group.
KC_HD inline void medoid_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    const uint32_t g0 = ch.mcount[r], g1 = ch.mcount[r + 1];
    if (g0 == g1) return;
    const int32_t F = (int32_t)ch.fcount[r], n = ch.n;
    const Tok *rt = ch.toks + (int64_t)ch.slot[r] * n;
    const uint32_t n_groups = ch.mcount[ch.R], n_strings = ch.scount[ch.R];
    for (int32_t j = lane; j < F; j += team) {
        const uint32_t d = ch.fdesc[ch.slot[r] + j];
        if (fdesc_kind(d) != F_MEDOID) continue;
        const Tok *row = rt + (int64_t)j * n;
        uint32_t live = 0;
        for (int32_t c = 0; c < n; ++c) live += row[c].kind != K_NULL ? 1u : 0u;
        if (live < 2) continue;
        const uint32_t g = g0 + fdesc_gidx(d);
        uint32_t s = ch.scount[r] + ch.piece_c[ch.slot[r] + j], at = ch.ccount[r] + ch.piece_l[ch.slot[r] + j];
        ch.mgrp_off[g] = (int32_t)s;
        for (int32_t c = 0; c < n; ++c) {
            if (row[c].kind == K_NULL) continue;
            ch.mstr_off[s++] = (int32_t)at;
            const uint8_t *v = ch.text + row[c].vstart;
            at += (row[c].flags & TOK_UNICODE) ? normalize_string(v, row[c].vlen, ch.mchars + at) : sanitized_copy(v, row[c].vlen, ch.mchars + at);
        }
        if (g + 1 == n_groups) {  // the chunk's last group closes both offset arrays
            ch.mgrp_off[n_groups] = (int32_t)n_strings;
            ch.mstr_off[n_strings] = (int32_t)at;
        }
    }
}

KC_HD inline void encode_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    if (load_status(ch, r)) return;
    const int32_t F = (int32_t)ch.fcount[r], n = ch.n;
    const Tok *rt = ch.toks + (int64_t)ch.slot[r] * n;
    for (int32_t j = lane; j < F; j += team) {
        const Tok *row = rt + (int64_t)j * n;
        const uint32_t d = ch.fdesc[ch.slot[r] + j], kind = fdesc_kind(d), g = fdesc_gidx(d);
        if (kind == F_VOTE_STR) {
            // local dictionary codes: the class of a cell is the first earlier cell with the same sanitised text
            int8_t *cells = ch.vcells + ((int64_t)ch.vbase[r] + g) * n;
            int32_t n_classes = 0;
            for (int32_t c = 0; c < n; ++c) {
                if (row[c].kind == K_NULL) {
                    cells[c] = (int8_t)KC_CODE_NONE;
                    continue;
                }
                int32_t code = -1;
                for (int32_t p = 0; p < c && code < 0; ++p)
                    if (row[p].kind != K_NULL && cells[p] >= 0 &&
                        sanitized_equal(ch.text + row[p].vstart, row[p].vlen, ch.text + row[c].vstart, row[c].vlen))
                        code = cells[p];
                cells[c] = (int8_t)(code >= 0 ? code : n_classes++);
            }
        } else if (kind == F_VOTE_BOOL) {
            int8_t *cells = ch.vcells + ((int64_t)ch.vbase[r] + g) * n;
            for (int32_t c = 0; c < n; ++c) cells[c] = row[c].kind == K_TRUE ? 1 : 0;  // None and False -> False (cu:956)
        } else if (kind == F_NUMERIC) {
            double *cells = ch.xcells + ((int64_t)ch.xbase[r] + g) * n;
            for (int32_t c = 0; c < n; ++c) {
                const Tok &t = row[c];
                double v;
                if (t.kind == K_NULL) {
                    v = bits_f64(KC_F64_NONE_BITS);
                } else if (t.kind == K_INT || t.kind == K_FLOAT) {
                    if (!to_double(ch.text + t.vstart, t.vlen, v)) {
                        decline(ch, r, D_NUMBER_RANGE);  // rows stay reserved; the emit phases skip the record
                        return;
                    }
                    if (t.kind == K_INT && v == 0.0) v = 0.0;  // int("-0") is 0: no negative zero from integers
                } else {
                    v = bits_f64(0x7FF8000000000000ull);  // bool / str: counted, never clustered
                }
                cells[c] = v;
            }
        }
    }
}

// ---------------------------------------------------------------- U1 - U3: the key-union round
//
// Record p of the round is plist[p].  After the pre-pass (cu:516-548) a missing key is an explicit None and a None (or missing)
// sub-object is an object of Nones at every level, so a record whose candidates differ in shape becomes a table of one shape:
// one row per key path of the union (depth-first, members in order of first appearance), a synthetic K_NULL where a candidate
// lacks the leaf, a synthetic K_OPEN / K_NULL... / K_CLOSE subtree where it lacks the object or holds None.  A1's type / order /
// slots / encode phases then run on that table unchanged.

KC_HD inline bool candidate_span(const Chunk &ch, int32_t r, int32_t c, int64_t &b, int64_t &len) {
    const int64_t base0 = ch.off[0];
    b = ch.off[(int64_t)r * ch.n + c] - base0;
    len = ch.off[(int64_t)r * ch.n + c + 1] - base0 - b;
    return len < ((int64_t)1 << 31) && b + len < ((int64_t)1 << 32);
}

// U1: lane c counts candidate c's tokens (scanning it afresh finds every scan-level reason to decline the record)
KC_HD inline void union_count_phase(const Chunk &ch, int32_t p, int32_t lane, int32_t team) {
    const int32_t r = ch.plist[p];
    for (int32_t c = lane; c < ch.n; c += team) {
        int64_t b, len;
        int32_t f = -D_TOO_LONG;
        if (candidate_span(ch, r, c, b, len)) f = scan_object(ch.text + b, (uint32_t)len, 0, nullptr, 0, kMaxFields, nullptr, false, nullptr, ch.unicode);
        if (f < 0) decline(ch, r, f == -D_TOO_MANY_FIELDS ? D_KEYS_DIFFER : -f);  // one candidate alone is over the union's limit
        ch.ucand[(int64_t)p * ch.n + c] = f > 0 ? (uint32_t)f : 0u;
    }
}

// U1, team leader: counts -> the candidates' first entries in the record's scratch region (entry 0: the root node), reserved
// from the chunk-wide counter
KC_HD inline void union_reserve(const Chunk &ch, int32_t p) {
    uint32_t *cand = ch.ucand + (int64_t)p * ch.n;
    uint32_t s = 1;
    for (int32_t c = 0; c < ch.n; ++c) {
        const uint32_t f = cand[c];
        cand[c] = s;
        s += f;
    }
    if (load_status(ch, ch.plist[p]) != D_UNION) s = 0;
    ch.usize[p] = s;
#ifdef __CUDA_ARCH__
    ch.ubase[p] = (uint32_t)atomicAdd(ch.counters + 4, (unsigned long long)s);
#else
    ch.ubase[p] = (uint32_t)ch.counters[4];
    ch.counters[4] += s;
#endif
}

// U2: lane c scans candidate c into the scratch region
KC_HD inline void union_scan_phase(const Chunk &ch, int32_t p, int32_t lane, int32_t team) {
    const int32_t r = ch.plist[p];
    if (load_status(ch, r) != D_UNION) return;
    for (int32_t c = lane; c < ch.n; c += team) {
        int64_t b, len;
        candidate_span(ch, r, c, b, len);  // U1 checked it
        scan_object(ch.text + b, (uint32_t)len, (uint32_t)b, ch.utok + ch.ubase[p] + ch.ucand[(int64_t)p * ch.n + c], 1, kMaxFields, nullptr, false,
                    nullptr, ch.unicode);
    }
}

KC_HD inline bool same_key(const Chunk &ch, const UNode &u, const Tok &t) {
    return u.klen == t.klen && key_compare(ch.text + u.kstart, u.klen, ch.text + t.kstart, t.klen) == 0;
}

// U2, team leader: the union tree, candidate by candidate.  A token's node is probed at the same position of the previous
// candidate, then after the node of its previous sibling, before the parent's members are searched: a reordered or one-key-
// short record costs about one more pass over its tokens.  Then the rows (depth-first) and the record's union slots.
KC_HD inline void union_build(const Chunk &ch, int32_t p) {
    const int32_t r = ch.plist[p], n = ch.n;
    if (load_status(ch, r) != D_UNION) return;
    const uint32_t base = ch.ubase[p], total = ch.usize[p];
    const uint32_t *cand = ch.ucand + (int64_t)p * n;
    const Tok *tk = ch.utok + base;
    UNode *nd = ch.unode + base;
    int32_t *map = ch.umap + base;
    nd[0] = UNode{0, 0, 0, 1, 0, -1, -1, -1, -1, -1, 0, 0};
    int32_t nn = 1;
    for (int32_t c = 0; c < n; ++c) {
        int32_t par[kMaxNesting + 2], sib[kMaxNesting + 2];  // per depth: the parent node, the node of the previous member
        par[0] = 0;
        sib[0] = -1;
        const uint32_t b = cand[c], e = c + 1 < n ? cand[c + 1] : total, pb = c ? cand[c - 1] : 0u;
        for (uint32_t i = b; i < e; ++i) {
            const Tok &t = tk[i];
            map[i] = -1;
            if (t.kind == K_CLOSE) continue;
            const uint32_t d = tok_depth(t);
            const int32_t P = par[d];
            int32_t u = -1;
            if (c > 0 && pb + (i - b) < b) {
                const int32_t v = map[pb + (i - b)];
                if (v > 0 && nd[v].parent == P && same_key(ch, nd[v], t)) u = v;
            }
            if (u < 0 && sib[d] > 0) {
                const int32_t v = nd[sib[d]].next;
                if (v > 0 && same_key(ch, nd[v], t)) u = v;
            }
            for (int32_t v = u < 0 ? nd[P].child : -1; v > 0; v = nd[v].next)
                if (same_key(ch, nd[v], t)) {
                    u = v;
                    break;
                }
            if (u < 0) {
                u = nn++;
                nd[u] = UNode{t.kstart, t.klen, (uint8_t)d, 0, 0, P, -1, -1, -1, -1, 0, 0};
                if (nd[P].last >= 0) nd[nd[P].last].next = u;
                else nd[P].child = u;
                nd[P].last = u;
            } else if (nd[u].lastc == c) {  // dict semantics would keep the last one: host path
                decline(ch, r, D_DUP_KEY);
                return;
            }
            nd[u].lastc = c;
            map[i] = u;
            if (t.kind == K_OPEN) {
                nd[u].obj = 1;
                par[d + 1] = u;
                sib[d + 1] = -1;
            } else if (t.kind != K_NULL) {
                nd[u].scalar = 1;
            }
            if (nd[u].obj && nd[u].scalar) {  // an object against a non-null value: the pre-pass leaves the values alone (cu:507-512)
                decline(ch, r, D_NESTED);
                return;
            }
            sib[d] = u;
        }
    }
    uint32_t rows = 0;
    uint8_t nested = 0;
    for (int32_t u = nd[0].child; u > 0;) {  // depth-first: an object's K_OPEN row, its members, its K_CLOSE row
        nd[u].row = rows++;
        nested |= nd[u].obj;
        if (nd[u].obj) {  // every object has a member: the scanner declines empty ones
            u = nd[u].child;
            continue;
        }
        while (u > 0 && nd[u].next < 0) {
            u = nd[u].parent;
            if (u > 0) nd[u].close = rows++;
        }
        if (u > 0) u = nd[u].next;
    }
    if (rows > (uint32_t)kMaxFields) {
        decline(ch, r, D_KEYS_DIFFER);
        return;
    }
    nd[0].row = (uint32_t)nn;
    ch.fcount[r] = rows;
    ch.nest[r] = nested;
#ifdef __CUDA_ARCH__
    ch.slot[r] = ch.uslot + (uint32_t)atomicAdd(ch.counters + 5, (unsigned long long)rows);
#else
    ch.slot[r] = ch.uslot + (uint32_t)ch.counters[5];
    ch.counters[5] += rows;
#endif
}

// U3: lane c writes column c of the [rows x n] table: synthetic tokens under every node (keyed like the node, so row 0 carries
// the key even where candidate 0 lacks it), then the candidate's own tokens over them (not its None where the node is an object)
KC_HD inline void union_write_phase(const Chunk &ch, int32_t p, int32_t lane, int32_t team) {
    const int32_t r = ch.plist[p], n = ch.n;
    if (load_status(ch, r) != D_UNION) return;
    const uint32_t base = ch.ubase[p];
    const uint32_t *cand = ch.ucand + (int64_t)p * n;
    const Tok *tk = ch.utok + base;
    const UNode *nd = ch.unode + base;
    const int32_t nn = (int32_t)nd[0].row;
    const int32_t *map = ch.umap + base;
    Tok *tab = ch.toks + (int64_t)ch.slot[r] * n;
    for (int32_t c = lane; c < n; c += team) {
        for (int32_t u = 1; u < nn; ++u) {
            Tok s;
            s.vstart = nd[u].kstart;
            s.vlen = 0;
            s.kstart = nd[u].kstart;
            s.klen = nd[u].klen;
            s.kind = nd[u].obj ? K_OPEN : K_NULL;
            s.flags = (uint8_t)(nd[u].depth << 4);
            tab[(int64_t)nd[u].row * n + c] = s;
            if (nd[u].obj) {
                s.kind = K_CLOSE;
                s.klen = 0;
                tab[(int64_t)nd[u].close * n + c] = s;
            }
        }
        const uint32_t e = c + 1 < n ? cand[c + 1] : ch.usize[p];
        for (uint32_t i = cand[c]; i < e; ++i) {
            const int32_t u = map[i];
            if (u < 0 || (nd[u].obj && tk[i].kind != K_OPEN)) continue;
            tab[(int64_t)nd[u].row * n + c] = tk[i];
        }
    }
}

// ---------------------------------------------------------------- C0 / C1

// one cell's original object as json.dumps prints it: ints keep their digits ("-0" is int 0), floats through float.__repr__
KC_HD inline void put_original(const Chunk &ch, const Tok &t, Sink &content) {
    if (t.kind == K_INT) {
        if (t.vlen == 2 && ch.text[t.vstart] == '-' && ch.text[t.vstart + 1] == '0') content.put('0');
        else content.put(ch.text + t.vstart, t.vlen);
    } else if (t.kind == K_FLOAT) {
        double v = 0.0;
        to_double(ch.text + t.vstart, t.vlen, v);
        float_repr(v, content);
    } else if (t.kind == K_STR) {
        content.json_string(ch.text + t.vstart, t.vlen, t.flags);
    } else {
        content.lit(t.kind == K_TRUE ? "true" : (t.kind == K_FALSE ? "false" : "null"));
    }
}

// value and confidence of one field, formatted into the two sinks (the epilogue emit_leaf of kc_json.cpp:
// cu:971-982, cu:1085-1086, cu:1116, cu:1177-1219); the confidences are kc::confidence / kc::medoid_confidence
KC_HD inline void format_field(const Chunk &ch, int32_t r, int32_t j, Sink &content, Sink &lik) {
    const int32_t n = ch.n;
    const Tok *row = ch.toks + ((int64_t)ch.slot[r] + j) * n;
    const uint32_t d = ch.fdesc[ch.slot[r] + j], kind = fdesc_kind(d), g = fdesc_gidx(d);
    double conf = 0.0;
    uint32_t m = 0;  // vote / numeric: the result word
    if (kind == F_VOTE_STR || kind == F_VOTE_BOOL) {
        m = ch.vmeta[(int64_t)ch.vbase[r] + g];
        const uint32_t idx = KC_META_IDX(m);
        if (kind == F_VOTE_BOOL) {
            content.lit(row[idx].kind == K_TRUE ? "true" : "false");  // the processed key (cu:958)
        } else {
            content.json_string(ch.text + row[idx].vstart, row[idx].vlen, row[idx].flags);  // first original whose sanitised form wins (cu:971)
        }
    } else if (kind == F_NUMERIC && ch.xmedoid) {  // the async dispatcher's similarity medoid (cu:1638-1688, K5)
        uint32_t live = 0;
        for (int32_t c = 0; c < n; ++c) live += row[c].kind != K_NULL ? 1u : 0u;
        const int64_t gi = (int64_t)ch.xbase[r] + g;
        int32_t want = ch.xbest[gi];
        conf = medoid_confidence(live, n, ch.xavg[gi]);
        for (int32_t c = 0; c < n; ++c) {
            if (row[c].kind == K_NULL) continue;
            if (want-- == 0) {
                put_original(ch, row[c], content);
                break;
            }
        }
    } else if (kind == F_NUMERIC) {
        m = ch.xmeta[(int64_t)ch.xbase[r] + g];
        const uint32_t idx = KC_META_IDX(m), flags = KC_META_FLAGS(m);
        if (flags & KC_FLAG_HAS_VALUE) {
            if (flags & KC_FLAG_SINGLE) {  // the original object, confidence unrounded (cu:1085-1086)
                put_original(ch, row[idx], content);
            } else {
                float_repr(ch.xvalue[(int64_t)ch.xbase[r] + g], content);
            }
        } else {
            content.lit("null");
        }
    } else if (kind == F_MEDOID) {
        uint32_t live = 0;
        for (int32_t c = 0; c < n; ++c) live += row[c].kind != K_NULL ? 1u : 0u;
        int32_t want = 0;  // one non-None string: itself
        double avg = 0.0;
        if (live >= 2) {
            const uint32_t gi = ch.mcount[r] + g;
            want = ch.midx[gi];
            avg = ch.mavg[gi];
        }
        conf = medoid_confidence(live, n, avg);
        for (int32_t c = 0; c < n; ++c) {
            if (row[c].kind == K_NULL) continue;
            if (want-- == 0) {
                content.json_string(ch.text + row[c].vstart, row[c].vlen, row[c].flags);
                break;
            }
        }
    } else {
        content.lit("null");  // all None: (None, 0.0) (cu:1401-1402)
    }
    // one call for both kinds keeps one inlined copy (two made write_kernel save convergence barriers); a vote group always
    // reaches the HAS_VALUE arm: a string group has a non-None cell, and a bool group turns None into False
    if (kind == F_VOTE_STR || kind == F_VOTE_BOOL || (kind == F_NUMERIC && !ch.xmedoid)) conf = confidence(m, kind == F_NUMERIC, 1.0);
    // likelihood-weighted calls: a vote leaf's likelihood is pvf (1 on this path) times K3b's weight share
    if (ch.vweight && (kind == F_VOTE_STR || kind == F_VOTE_BOOL)) conf = weighted_vote_confidence(1.0, ch.vweight[(int64_t)ch.vbase[r] + g]);
    float_repr(conf, lik);
}

KC_HD inline void len_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    if (load_status(ch, r)) return;
    const int32_t F = (int32_t)ch.fcount[r], n = ch.n;
    for (int32_t j = lane; j < F; j += team) {
        const uint32_t d = ch.fdesc[ch.slot[r] + j], kind = fdesc_kind(d), sep = fdesc_last(d) ? 0u : 2u;  // ", " unless last of its siblings
        const Tok &t0 = ch.toks[((int64_t)ch.slot[r] + j) * n];
        const uint32_t head = (t0.flags & TOK_ELEM) ? 0u : t0.klen + 4u;  // "key": (a list element has no key)
        const uint32_t pos = out_pos(ch, r, j);
        uint32_t lc, ll;
        if (kind == F_OPEN || kind == F_LOPEN) {
            lc = ll = head + 1u;  // "key": {   "key": [
        } else if (kind == F_CLOSE || kind == F_LCLOSE) {
            lc = ll = 1u + sep;   // }   ]
        } else {
            Sink c{nullptr, 0}, l{nullptr, 0};
            format_field(ch, r, j, c, l);
            lc = head + (uint32_t)c.n + sep;  // "key": value
            ll = head + (uint32_t)l.n + sep;
        }
        ch.piece_c[ch.slot[r] + pos] = lc;
        ch.piece_l[ch.slot[r] + pos] = ll;
    }
}

// team leader only: piece lengths (in key order) -> piece offsets; record lengths
KC_HD inline void offsets_phase(const Chunk &ch, int32_t r) {
    if (load_status(ch, r)) {
        ch.len_c[r] = 0;
        ch.len_l[r] = 0;
        return;
    }
    const int32_t F = (int32_t)ch.fcount[r];
    uint32_t *pc = ch.piece_c + ch.slot[r], *pl = ch.piece_l + ch.slot[r];
    uint32_t oc = 1, ol = 1;  // after '{'
    for (int32_t k = 0; k < F; ++k) {  // pieces in output order, separators included
        const uint32_t lc = pc[k], ll = pl[k];
        pc[k] = oc;
        pl[k] = ol;
        oc += lc;
        ol += ll;
    }
    ch.len_c[r] = (int64_t)oc + 1;  // '}'
    ch.len_l[r] = (int64_t)ol + 1;
}

KC_HD inline void write_phase(const Chunk &ch, int32_t r, int32_t lane, int32_t team) {
    if (load_status(ch, r)) return;
    const int32_t F = (int32_t)ch.fcount[r], n = ch.n;
    uint8_t *oc = ch.out_c + ch.len_c[r], *ol = ch.out_l + ch.len_l[r];  // len_* hold the scanned offsets now
    for (int32_t j = lane; j < F; j += team) {
        const Tok &t0 = ch.toks[((int64_t)ch.slot[r] + j) * n];
        const uint32_t d = ch.fdesc[ch.slot[r] + j], kind = fdesc_kind(d);
        const uint32_t pos = out_pos(ch, r, j);
        Sink c{oc + ch.piece_c[ch.slot[r] + pos], 0}, l{ol + ch.piece_l[ch.slot[r] + pos], 0};
        if (pos == 0) {
            oc[0] = '{';
            ol[0] = '{';
        }
        if (kind == F_CLOSE || kind == F_LCLOSE) {
            const uint8_t b = kind == F_CLOSE ? '}' : ']';
            c.put(b);
            l.put(b);
        } else {
            if (!(t0.flags & TOK_ELEM)) {
                c.put('"');
                c.put(ch.text + t0.kstart, t0.klen);
                c.lit("\": ");
                l.put('"');
                l.put(ch.text + t0.kstart, t0.klen);
                l.lit("\": ");
            }
            if (kind == F_OPEN || kind == F_LOPEN) {
                const uint8_t b = kind == F_OPEN ? '{' : '[';
                c.put(b);
                l.put(b);
                continue;
            }
            format_field(ch, r, j, c, l);
        }
        if (!fdesc_last(d)) {
            c.lit(", ");
            l.lit(", ");
        } else if (tok_depth(t0) == 0) {  // the last piece of the record closes the top-level object
            c.put('}');
            l.put('}');
        }
    }
}

// ---------------------------------------------------------------- steps: each kernel's schedule of phases
//
// A step runs the phases of one unit of work (a record; in the union round, record plist[p]) on a team, in the kernel's order.
// On the device a team is `size` lanes of one warp: a phase runs on the lanes of a live team, then the whole warp meets at
// __syncwarp() (which also orders the team's global-memory traffic between phases).  A dead team (no unit left this round)
// still reaches every __syncwarp() of the live teams of its warp.  On the host a team is a loop over its lanes.

struct DeviceTeam {
    int32_t lane, size;
    bool live;
    KC_HD void sync() const {
#ifdef __CUDA_ARCH__
        __syncwarp();
#endif
    }
    template <class F>
    KC_HD void each(const F &f) const {
        if (live) f(lane);
        sync();
    }
    template <class F>
    KC_HD void leader(const F &f) const {
        if (live && lane == 0) f();
        sync();
    }
    // a kernel's only phase: no lane reads what another one wrote, so the lanes need not meet
    template <class F>
    KC_HD void each_nosync(const F &f) const {
        if (live) f(lane);
    }
};

struct HostTeam {
    int32_t size;
    static constexpr bool live = true;
    template <class F>
    KC_HD void each(const F &f) const {
        for (int32_t lane = 0; lane < size; ++lane) f(lane);
    }
    template <class F>
    KC_HD void leader(const F &f) const { f(); }
    template <class F>
    KC_HD void each_nosync(const F &f) const { each(f); }
};

// A1 after the parse, and U3 after the table: type / order / slots / encode
template <class Team>
KC_HD void table_phases(const Chunk &ch, int32_t r, const Team &tm, bool first_round) {
    tm.each([&](int32_t lane) { type_phase(ch, r, lane, tm.size); });
    tm.each([&](int32_t lane) { order_phase(ch, r, lane, tm.size); });  // nested records only; reads the ranks its team wrote
    tm.leader([&] { slots_phase(ch, r, first_round); });
    tm.each([&](int32_t lane) { encode_phase(ch, r, lane, tm.size); });
}

template <class Team>
KC_HD void plan_step(const Chunk &ch, int32_t r, const Team &tm) {
    tm.each([&](int32_t lane) { parse_phase(ch, r, lane, tm.size); });
    table_phases(ch, r, tm, true);
}

template <class Team>
KC_HD void union_count_step(const Chunk &ch, int32_t p, const Team &tm) {
    tm.each([&](int32_t lane) { union_count_phase(ch, p, lane, tm.size); });
    tm.leader([&] { union_reserve(ch, p); });
}

template <class Team>
KC_HD void union_build_step(const Chunk &ch, int32_t p, const Team &tm) {
    tm.each([&](int32_t lane) { union_scan_phase(ch, p, lane, tm.size); });
    tm.leader([&] { union_build(ch, p); });
}

// the table, then A1's phases on it (the leader clears the status between the two)
template <class Team>
KC_HD void union_plan_step(const Chunk &ch, int32_t p, const Team &tm) {
    const int32_t r = tm.live ? ch.plist[p] : 0;
    tm.each([&](int32_t lane) { union_write_phase(ch, p, lane, tm.size); });
    tm.leader([&] {
        if (load_status(ch, r) == D_UNION) decline(ch, r, D_OK);
    });
    table_phases(ch, r, tm, false);
}

template <class Team>
KC_HD void medoid_step(const Chunk &ch, int32_t r, const Team &tm) {
    tm.each_nosync([&](int32_t lane) { medoid_phase(ch, r, lane, tm.size); });
}

template <class Team>
KC_HD void len_step(const Chunk &ch, int32_t r, const Team &tm) {
    tm.each([&](int32_t lane) { len_phase(ch, r, lane, tm.size); });
    tm.leader([&] { offsets_phase(ch, r); });
}

template <class Team>
KC_HD void write_step(const Chunk &ch, int32_t r, const Team &tm) {
    tm.each_nosync([&](int32_t lane) { write_phase(ch, r, lane, tm.size); });
}

// ---------------------------------------------------------------- kernels

#ifdef __CUDACC__

__global__ void __launch_bounds__(128) count_kernel(const Chunk ch) {
    for (int32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < ch.R; r += gridDim.x * blockDim.x) count_record(ch, r);
}

// Team t of a warp owns unit (warp_index * teams_per_warp + t) of every grid-stride round; all lanes of the warp walk the
// same rounds, so they meet at the same __syncwarp()s.
template <class Step>
__device__ __forceinline__ void team_loop(int32_t team, int64_t units, const Step &step) {
    const int32_t lane_w = threadIdx.x & 31, tpw = 32 / team;
    const int32_t lane = lane_w % team, t = lane_w / team;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t rounds = (units + tpw - 1) / tpw;
    for (int64_t w = warp; w < rounds; w += n_warps) {
        const int64_t u = w * tpw + t;
        step((int32_t)u, DeviceTeam{lane, team, u < units});
    }
}

__global__ void __launch_bounds__(128) plan_kernel(const Chunk ch, int32_t team) {
    team_loop(team, ch.R, [&](int32_t r, const DeviceTeam &tm) { plan_step(ch, r, tm); });
}

__global__ void __launch_bounds__(128) union_count_kernel(const Chunk ch, int32_t team, int32_t P) {
    team_loop(team, P, [&](int32_t p, const DeviceTeam &tm) { union_count_step(ch, p, tm); });
}

__global__ void __launch_bounds__(128) union_build_kernel(const Chunk ch, int32_t team, int32_t P) {
    team_loop(team, P, [&](int32_t p, const DeviceTeam &tm) { union_build_step(ch, p, tm); });
}

__global__ void __launch_bounds__(128) union_plan_kernel(const Chunk ch, int32_t team, int32_t P) {
    team_loop(team, P, [&](int32_t p, const DeviceTeam &tm) { union_plan_step(ch, p, tm); });
}

__global__ void __launch_bounds__(128) medoid_kernel(const Chunk ch, int32_t team) {
    team_loop(team, ch.R, [&](int32_t r, const DeviceTeam &tm) { medoid_step(ch, r, tm); });
}

__global__ void __launch_bounds__(128) len_kernel(const Chunk ch, int32_t team) {
    team_loop(team, ch.R, [&](int32_t r, const DeviceTeam &tm) { len_step(ch, r, tm); });
}

__global__ void __launch_bounds__(128) write_kernel(const Chunk ch, int32_t team) {
    team_loop(team, ch.R, [&](int32_t r, const DeviceTeam &tm) { write_step(ch, r, tm); });
}

#endif  // __CUDACC__

}  // namespace js
}  // namespace kc
