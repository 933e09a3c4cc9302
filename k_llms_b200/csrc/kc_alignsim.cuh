// kc_alignsim.cuh — element similarities of the list-alignment pre-pass (H2) for a batch of list nodes.
//
// lists_alignment (cu:185-430) compares list elements pairwise through generic_similarity (cu:892-917), memoised in a
// dense T x T matrix per list node (kc_align.inl, ListAligner).  This phase fills that matrix ahead of the alignment for
// the elements it can model, bit for bit as the host computes them:
//   - `not bool(v)` on both sides -> 1.0; None on one side -> the 1e-8 floor;
//   - bool / int / float: numerical_similarity (cu:827-841), math.isclose with rel_tol = 0.01;
//   - strings: raw-equal -> 1.0; both normalised forms empty -> 1.0; else 1 - d / longest (one IEEE division, floored at
//     1e-8) with d the edit distance of the normalised forms: Myers' bit-parallel algorithm with K4's match tables and inner
//     loop (kc_medoid.cuh), the shorter form as the pattern;
//   - flat dicts (scalar or None values): the member similarities over the union of keys in SORTED key order (the keys
//     reasoning___* / source___* skipped, a missing key is None), summed from 0.0 and divided once.
// Every other pair is left NaN ("not computed") and the host computes it lazily if the alignment asks for it:
//   - two strings both longer than 50 raw characters (the reference sends them to the embeddings service, cu:813: the host's
//     string_similarity marks the record for the Python path, and only if that pair is needed);
//   - strings whose shorter normalised form is longer than 64 characters (one 64-bit Myers word);
//   - lists, dicts holding dicts or lists, and pairs of different shapes (string / number / dict).
// The diagonal stays NaN as well: the alignment never compares an element with itself.
//
// One warp per node, lanes over the pairs a < b; each lane builds the match table of its pair's pattern in its own slice
// of shared memory.  The phase functions are __host__ __device__ on plain arrays: kc_alignsim(device < 0) runs the same
// source on the host, which is what the CPU tests check.
#pragma once

#include "kc_internal.h"  // py_isclose, kSimFloor
#include "kc_medoid.cuh"  // alnum_index, myers_table, myers, kAlphabet, kPeqStride

namespace kc {

constexpr int kAlignSimMaxT = 512;        // the host's dense memo limit (ListAligner)
constexpr int kAlignSimMaxPattern = 64;   // the shorter normalised string of a pair must fit one 64-bit word
constexpr int kAlignSimEmbedLen = 50;     // both raw strings longer than this: embeddings pair (cu:813)

__host__ __device__ __forceinline__ double alignsim_nan() {
    const uint64_t bits = 0x7FF8000000000000ull;
    double d;
    memcpy(&d, &bits, 8);
    return d;
}

// generic_similarity of two scalars (or None); tab: the lane's match table (kPeqStride u64)
__host__ __device__ inline double alignsim_value(const KcAsVal &x, const KcAsVal &y, const uint8_t *__restrict__ chars, uint64_t *tab) {
    if ((x.flags & y.flags & KC_AS_FALSY) != 0) return 1.0;
    if (x.type == KC_AS_NONE || y.type == KC_AS_NONE) return kSimFloor;
    if (x.type == KC_AS_STR && y.type == KC_AS_STR) {  // string_similarity, cu:797-824
        if (x.raw_len > kAlignSimEmbedLen && y.raw_len > kAlignSimEmbedLen) return alignsim_nan();
        if (x.raw_id == y.raw_id) return 1.0;
        const bool xs = x.len <= y.len;
        const KcAsVal &p = xs ? x : y, &t = xs ? y : x;  // pattern = the shorter normalised form
        if (t.len == 0) return 1.0;
        if (p.len > kAlignSimMaxPattern) return alignsim_nan();
        int d;
        if (p.len == 0) {
            d = t.len;
        } else {
            myers_table(tab, chars + p.off, p.len);
            d = p.len <= 32 ? myers<uint32_t>(tab, p.len, chars + t.off, t.len) : myers<uint64_t>(tab, p.len, chars + t.off, t.len);
        }
        const double sim = 1.0 - (double)d / (double)t.len;
        return sim > kSimFloor ? sim : kSimFloor;
    }
    const bool xn = x.type == KC_AS_BOOL || x.type == KC_AS_INT || x.type == KC_AS_FLOAT;
    const bool yn = y.type == KC_AS_BOOL || y.type == KC_AS_INT || y.type == KC_AS_FLOAT;
    if (xn && yn) {  // numerical_similarity, cu:827-841
        if (x.type == KC_AS_BOOL && y.type == KC_AS_BOOL) return x.num == y.num ? 1.0 : kSimFloor;
        if (py_isclose(x.num, y.num)) return 1.0;
        // int vs int compares the decimal texts: equal canonical keys (texts that fit int64) are equal texts
        const bool eq = (x.type == KC_AS_INT && y.type == KC_AS_INT) ? (x.ikey == y.ikey && ((x.flags | y.flags) & KC_AS_BIGINT) == 0)
                                                                    : x.num == y.num;
        return eq ? 1.0 : kSimFloor;
    }
    return alignsim_nan();  // lists, nested dicts, mixed shapes: the host's
}

// generic_similarity of two list elements
__host__ __device__ inline double alignsim_pair(const KcAsVal &x, const KcAsVal &y, const KcAsVal *__restrict__ vals,
                                                const uint8_t *__restrict__ chars, uint64_t *tab) {
    if (x.type == KC_AS_DICT && y.type == KC_AS_DICT && (x.flags & y.flags & KC_AS_FALSY) == 0) {  // cu:844-869
        KcAsVal none{};
        none.type = KC_AS_NONE;
        none.flags = KC_AS_FALSY;
        const KcAsVal *p = vals + x.off, *q = vals + y.off;
        int i = 0, j = 0, keys = 0;
        double total = 0.0;
        while (i < x.len || j < y.len) {  // merge of the two sorted member lists = the sorted union of the keys
            double s;
            if (j >= y.len || (i < x.len && p[i].key < q[j].key)) s = alignsim_value(p[i++], none, chars, tab);
            else if (i >= x.len || q[j].key < p[i].key) s = alignsim_value(none, q[j++], chars, tab);
            else s = alignsim_value(p[i++], q[j++], chars, tab);
            total += s;  // a NaN member makes the whole pair NaN: the host computes it
            ++keys;
        }
        return keys == 0 ? 1.0 : total / (double)keys;
    }
    return alignsim_value(x, y, chars, tab);
}

// The matrix of one node, pairs a < b split over `lanes` lanes.  Returns the pairs this lane decided (not NaN).
__host__ __device__ inline int64_t alignsim_node(const KcAsNode &nd, const KcAsVal *__restrict__ vals, const uint8_t *__restrict__ chars,
                                                 double *__restrict__ out, int lane, int lanes, uint64_t *tab) {
    const int T = nd.T;
    const KcAsVal *e = vals + nd.val0;
    double *m = out + nd.out;
    for (int i = lane; i < T; i += lanes) m[(size_t)i * T + i] = alignsim_nan();
    int64_t decided = 0;
    int a = 0, b = 1 + lane;  // (a, b) walks the upper triangle row by row, `lanes` pairs at a time
    while (a < T - 1 && b >= T) {
        const int over = b - T;
        ++a;
        b = a + 1 + over;
    }
    while (a < T - 1) {
        const double s = alignsim_pair(e[a], e[b], vals, chars, tab);
        m[(size_t)a * T + b] = s;
        m[(size_t)b * T + a] = s;
        decided += s == s;
        b += lanes;
        while (a < T - 1 && b >= T) {
            const int over = b - T;
            ++a;
            b = a + 1 + over;
        }
    }
    return decided;
}

#ifdef __CUDACC__
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) alignsim_kernel(const KcAsNode *__restrict__ nodes, int64_t n_nodes,
                                                              const KcAsVal *__restrict__ vals, const uint8_t *__restrict__ chars,
                                                              double *__restrict__ out, unsigned long long *__restrict__ pairs) {
    __shared__ uint64_t tabs[WARPS * 32 * kPeqStride];  // one match table per lane (odd stride: lanes spread over the banks)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t *tab = tabs + (size_t)threadIdx.x * kPeqStride;
    int64_t decided = 0;
    for (int64_t g = (int64_t)blockIdx.x * WARPS + warp; g < n_nodes; g += (int64_t)gridDim.x * WARPS)
        decided += alignsim_node(nodes[g], vals, chars, out, lane, 32, tab);
#pragma unroll
    for (int st = 16; st >= 1; st >>= 1) decided += __shfl_xor_sync(0xFFFFFFFFu, decided, st);
    if (lane == 0 && decided) atomicAdd(pairs, (unsigned long long)decided);
}
#endif

}  // namespace kc
