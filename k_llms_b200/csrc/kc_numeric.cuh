// kc_numeric.cuh — K2: numeric consensus.  One thread owns one group of n float64 cells.
//
// Replaces the numeric branch of consensus_as_primitive (reference consensus_utils.py:1098-1219):
//   sort -> chain adjacent values closer than max(abs_eps, rel_eps*max(|a|,|b|,1)) into clusters (cu:1127-1144)
//   -> unique largest cluster: float(np.mean(cluster)), support = size            (cu:1171-1187)
//   -> tie: neighbours' support, then (spread, -|center|) ordering                (cu:1189-1219)
// Bit-exactness: np.mean / np.std are numpy pairwise sums (8 accumulators, (r0+r1)+(r2+r3)+..., tail
// left-to-right, reduction seeded with +0.0); every add/mul/div/sqrt below is a single IEEE-754
// round-to-nearest operation in that order (the file is compiled with -fmad=false as well).
//
// Cost model: the op is HBM-streaming (8n bytes in, 12 out per group) but a 64-bit sort in 32-bit registers is
// select-bound, so the sort runs on 32-bit KEYS instead: the order-preserving image of each cell's high word
// with the candidate index in the low log2(n) bits.  A compare-exchange is then one IMNMX pair.  The cells
// themselves stay in shared memory ("row memory": a [cell][thread] plane) and are fetched once in key order.
// Keys drop the low mantissa bits, so values that differ only there may come out swapped; a 15-compare
// sortedness check detects that and a shared-memory insertion sort of the (rare) offending row repairs it.
// Non-finite cells get keys above every finite key and sort to the end.
#pragma once

#include <type_traits>
#include <utility>

#include "kc_common.cuh"
#include "kc_csa.cuh"
#include "kc_vote.cuh"  // MaskOf, popc_m

namespace kc {

constexpr uint32_t kNoneHi = (uint32_t)(KC_F64_NONE_BITS >> 32);      // only the HIGH word of a cell tags it
constexpr uint32_t kAbsentHi = (uint32_t)(KC_F64_ABSENT_BITS >> 32);
constexpr uint32_t kKeyNonFinite = 0xFFE00000u;  // keys >= this belong to non-finite cells

__device__ __forceinline__ int ffs_m(uint32_t m) { return __ffs((int)m); }
__device__ __forceinline__ int ffs_m(uint64_t m) { return __ffsll((long long)m); }
__device__ __forceinline__ int clz_m(uint32_t m) { return __clz((int)m); }
__device__ __forceinline__ int clz_m(uint64_t m) { return __clzll((long long)m); }

// 10.0**k for k = -6..6 exactly as CPython computes it (correctly rounded decimal literals): cu:1156-1157.
__device__ __constant__ double kPow10[13] = {1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6};

// ---------------------------------------------------------------- row memory

__device__ __forceinline__ double lds_f64(uint32_t addr) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_f64(uint32_t addr, double v) {
    asm volatile("st.shared.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
__device__ __forceinline__ uint2 lds_u32x2(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}

struct PlaneRow {  // [cell][thread] plane: pitch = threads*8 bytes, a multiple of 128 => bank depends on tid only
    uint32_t base, pitch;
    __device__ __forceinline__ uint32_t addr(uint32_t elem) const { return base + elem * pitch; }
    // same address as one IMAD (FMA pipe) instead of shift + add on the busier ALU pipe
    __device__ __forceinline__ uint32_t addr_mad(uint32_t elem) const {
        uint32_t a;
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(elem), "r"(pitch), "r"(base));
        return a;
    }
};

// ---------------------------------------------------------------- row loader: cells 2q and 2q+1 arrive as one 16-byte load

// the 2Q cells at p (one row, or several small rows) as Q 16-byte loads
template <int Q>
__device__ __forceinline__ void load_cells(const double *p, int4 (&c)[Q]) {
#pragma unroll
    for (int q = 0; q < Q; ++q) c[q] = ldg_nc_v4(reinterpret_cast<const int4 *>(p) + q);
}

// grid-stride over units u < n_units: the next unit is requested before body(u, cells) works on this one
template <int Q, class Body>
__device__ __forceinline__ void prefetch_units(const double *vals, int64_t u, int64_t n_units, int64_t stride, Body body) {
    int4 cur[Q];
    if (u < n_units) load_cells(vals + u * (2 * Q), cur);
    for (; u < n_units; u += stride) {
        int4 nxt[Q];
        if (u + stride < n_units) load_cells(vals + (u + stride) * (2 * Q), nxt);
        body(u, cur);
#pragma unroll
        for (int q = 0; q < Q; ++q) cur[q] = nxt[q];
    }
}

__device__ __forceinline__ void put_pair(const PlaneRow row, int q, int4 c) {
    sts_f64(row.addr(2 * q + 0), __hiloint2double(c.y, c.x));
    sts_f64(row.addr(2 * q + 1), __hiloint2double(c.w, c.z));
}

// numeric_core's input: the high words in hi[], the cells in the plane
template <int N>
__device__ __forceinline__ void load_pair(int4 c, int q, uint32_t (&hi)[N], const PlaneRow row) {
    hi[2 * q + 0] = (uint32_t)c.y;
    hi[2 * q + 1] = (uint32_t)c.w;
    put_pair(row, q, c);
}

// the high words of a row parked in the plane
template <int N>
__device__ __forceinline__ void plane_hi(const PlaneRow row, uint32_t (&hi)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) hi[i] = lds_u32x2(row.addr(i)).y;
}

// ---------------------------------------------------------------- numpy reductions over sorted row memory

// numpy DOUBLE_pairwise_sum (n <= 128) over f(0..n-1), then the +0.0 seed of add.reduce.
template <typename F>
__device__ __forceinline__ double np_sum(F f, int n) {
    double res;
    if (n < 8) {
        res = -0.0;
        for (int i = 0; i < n; ++i) res = __dadd_rn(res, f(i));
    } else {
        double r0 = f(0), r1 = f(1), r2 = f(2), r3 = f(3), r4 = f(4), r5 = f(5), r6 = f(6), r7 = f(7);
        int i = 8;
        const int n8 = n - (n & 7);
        for (; i < n8; i += 8) {
            r0 = __dadd_rn(r0, f(i + 0));
            r1 = __dadd_rn(r1, f(i + 1));
            r2 = __dadd_rn(r2, f(i + 2));
            r3 = __dadd_rn(r3, f(i + 3));
            r4 = __dadd_rn(r4, f(i + 4));
            r5 = __dadd_rn(r5, f(i + 5));
            r6 = __dadd_rn(r6, f(i + 6));
            r7 = __dadd_rn(r7, f(i + 7));
        }
        res = __dadd_rn(__dadd_rn(__dadd_rn(r0, r1), __dadd_rn(r2, r3)), __dadd_rn(__dadd_rn(r4, r5), __dadd_rn(r6, r7)));
        for (; i < n; ++i) res = __dadd_rn(res, f(i));
    }
    return __dadd_rn(0.0, res);
}

template <typename Row>
__device__ __forceinline__ double np_mean(const Row &xs, int s, int len) {
    return __ddiv_rn(np_sum([&](int i) { return lds_f64(xs.addr(s + i)); }, len), (double)len);
}

// The same sum for groups of at most 16 cells, without data-dependent loops: fewer than 8 terms -> up to 7
// predicated adds; otherwise 8 accumulators (two terms each only when all 16 cells are in the cluster), the tree, and
// up to 7 predicated tail adds.
template <typename Row>
__device__ __forceinline__ double np_mean16(const Row &xs, int s, int len) {
    const uint32_t a0 = xs.addr_mad((uint32_t)s);
    const uint32_t pitch = xs.addr(1) - xs.addr(0);
    double res;
    if (len < 8) {
        res = -0.0;
#pragma unroll
        for (int j = 0; j < 7; ++j)
            if (j < len) res = __dadd_rn(res, lds_f64(a0 + j * pitch));
    } else {
        double r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = lds_f64(a0 + j * pitch);
        int tail = 8;
        if (len >= 16) {
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], lds_f64(a0 + (8 + j) * pitch));
            tail = 16;
        }
        res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                        __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
#pragma unroll
        for (int j = 0; j < 7; ++j)
            if (tail + j < len) res = __dadd_rn(res, lds_f64(a0 + (tail + j) * pitch));
    }
    return __ddiv_rn(__dadd_rn(0.0, res), (double)len);
}

template <typename Row>
__device__ __forceinline__ double np_median(const Row &xs, int s, int len) {  // ascending input
    if (len & 1) return __dadd_rn(0.0, __dadd_rn(-0.0, lds_f64(xs.addr(s + len / 2))));
    return __ddiv_rn(
        __dadd_rn(0.0, __dadd_rn(__dadd_rn(-0.0, lds_f64(xs.addr(s + len / 2 - 1))), lds_f64(xs.addr(s + len / 2)))), 2.0);
}

template <typename Row>
__device__ __forceinline__ double np_std(const Row &xs, int s, int len) {
    const double mean = np_mean(xs, s, len);
    const double ss = np_sum(
        [&](int i) {
            const double d = __dadd_rn(lds_f64(xs.addr(s + i)), -mean);
            return __dmul_rn(d, d);
        },
        len);
    return __dsqrt_rn(__ddiv_rn(ss, (double)len));
}

__device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }  // NaN-free operands only

__device__ __forceinline__ bool is_close(double a, double b, double rel_eps, double abs_eps) {  // cu:1146-1148
    const double denom = dmax(dmax(fabs(a), fabs(b)), 1.0);
    return fabs(__dadd_rn(a, -b)) <= dmax(abs_eps, __dmul_rn(rel_eps, denom));
}

__device__ __forceinline__ bool is_close_pow10(double a, double b, double rel_eps, double abs_eps) {  // cu:1153-1160
    if (a == 0.0 || b == 0.0) return is_close(a, b, rel_eps, abs_eps);
    for (int k = 0; k < 13; ++k)
        if (is_close(a, __dmul_rn(b, kPow10[k]), rel_eps, abs_eps)) return true;
    return false;
}

struct TieResult {
    double value;
    int support;
};

// Tie between equally large clusters (cu:1189-1219).  `starts` has one bit per cluster start (< m).
template <typename M, typename Row>
__device__ __noinline__ TieResult numeric_tie(const Row xs, M starts, int m, int top, double rel_eps, double abs_eps) {
    int best_s = -1, best_support = 0;
    double best_spread = 0.0, best_center = 0.0;
    M sk = starts;
    while (sk) {
        const int s = ffs_m(sk) - 1;
        sk &= sk - 1;
        const int e = sk ? ffs_m(sk) - 1 : m;
        const int len = e - s;
        if (len != top) continue;
        const double center = np_median(xs, s, len);
        int support = top;
        M so = starts;
        while (so) {
            const int os = ffs_m(so) - 1;
            so &= so - 1;
            const int oe = so ? ffs_m(so) - 1 : m;
            const int olen = oe - os;
            if (olen >= top) continue;  // only strictly smaller clusters lend support (cu:1200)
            const double oc = np_median(xs, os, olen);
            if (is_close(center, oc, rel_eps, abs_eps) || is_close(fabs(center), fabs(oc), rel_eps, abs_eps) ||
                is_close_pow10(center, oc, rel_eps, abs_eps))
                support += olen;
        }
        const double spread = len > 1 ? np_std(xs, s, len) : 0.0;
        // sort key (-support, spread, -|center|), stable (cu:1211): only a strict improvement replaces the best
        const bool better = best_s < 0 || support > best_support ||
                            (support == best_support &&
                             (spread < best_spread || (spread == best_spread && fabs(center) > fabs(best_center))));
        if (better) {
            best_s = s;
            best_support = support;
            best_spread = spread;
            best_center = center;
        }
    }
    return TieResult{np_mean(xs, best_s, top), best_support};
}

// ---------------------------------------------------------------- 32-bit key sort

// Batcher merge-exchange network, ascending, N a power of two; comparator list built at compile time and
// expanded as a fold so every register index is a constant.
template <int N>
struct BatcherNet {
    int a[N * N / 2 + 1];
    int b[N * N / 2 + 1];
    int count;
    constexpr BatcherNet() : a{}, b{}, count(0) {
        for (int p = 1; p < N; p *= 2)
            for (int k = p; k >= 1; k /= 2)
                for (int j = k % p; j <= N - 1 - k; j += 2 * k)
                    for (int i = 0; i < k; ++i)
                        if (i + j + k < N && (i + j) / (2 * p) == (i + j + k) / (2 * p)) {
                            a[count] = i + j;
                            b[count] = i + j + k;
                            ++count;
                        }
    }
};

template <int A, int B, int N>
__device__ __forceinline__ void compare_exchange(uint32_t (&x)[N]) {
    const uint32_t lo = min(x[A], x[B]), hi = max(x[A], x[B]);
    x[A] = lo;
    x[B] = hi;
}

template <int N, size_t... I>
__device__ __forceinline__ void sort_keys_impl(uint32_t (&x)[N], std::index_sequence<I...>) {
    constexpr BatcherNet<N> net{};
    (compare_exchange<net.a[I], net.b[I], N>(x), ...);
}

template <int N>
__device__ __forceinline__ void sort_keys(uint32_t (&x)[N]) {
    constexpr BatcherNet<N> net{};
    sort_keys_impl<N>(x, std::make_index_sequence<net.count>{});
}

// `bit` unless d <= p or d <= q or d <= thr (ordered compares: NaN -> not close).  Written in PTX so the three
// tests stay three predicate-combining DSETPs; left to the optimiser they turn into fmax() expansions.
__device__ __forceinline__ uint32_t far_bit(double d, double p, double q, double thr, uint32_t bit) {
    uint32_t r;
    asm("{\n\t"
        ".reg .pred c;\n\t"
        "setp.le.f64 c, %1, %2;\n\t"
        "setp.le.or.f64 c, %1, %3, c;\n\t"
        "setp.le.or.f64 c, %1, %4, c;\n\t"
        "selp.u32 %0, 0, %5, c;\n\t"
        "}"
        : "=r"(r)
        : "d"(d), "d"(p), "d"(q), "d"(thr), "r"(bit));
    return r;
}

// Insertion sort of row[0..m) (finite values) — only reached when two distinct values share a truncated key.
template <typename Row>
__device__ __noinline__ void repair_sorted_prefix(const Row row, int m) {
    for (int i = 1; i < m; ++i) {
        const double v = lds_f64(row.addr(i));
        int j = i - 1;
        while (j >= 0) {
            const double u = lds_f64(row.addr(j));
            if (!(u > v)) break;
            sts_f64(row.addr(j + 1), u);
            --j;
        }
        sts_f64(row.addr(j + 1), v);
    }
}

// ---------------------------------------------------------------- the core

// hi[i] = high word of raw cell i; the raw cells are also resident in `row` (cell i at row.addr(i)).
// On return row memory holds the sorted finite values (scratch).  thr = max(abs_eps, rel_eps*1.0).
template <int N, typename Row>
__device__ __forceinline__ void numeric_core(const uint32_t (&hi)[N], const Row row, double rel_eps, double abs_eps,
                                             double thr, double &value, uint32_t &meta) {
    using M = typename MaskOf<N>::type;
    static_assert(N >= 2 && (N & (N - 1)) == 0, "N must be a power of two >= 2");
    constexpr uint32_t IDX = N - 1;
    const double qnan = __longlong_as_double(0x7FF8000000000000LL);

    // A. keys and the cell census.  t is a bijective, order-preserving image of the high word; z = t - 0xFFE00000 is
    //    < 0x200000 exactly for non-finite cells, and the two tags are adjacent high words, so u = z - Z_NONE is
    //    0 (None) or 1 (absent) for tagged cells.  One packed counter (tagged << 16 | nonfinite << 8 | absent) takes
    //    a single add per cell.
    constexpr uint32_t Z_NONE = ((kNoneHi ^ 0x80000000u) - 0x00100000u) - kKeyNonFinite;
    static_assert(kAbsentHi == kNoneHi + 1, "tags must be adjacent high words");
    uint32_t key[N];
    uint32_t census = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const uint32_t s = (uint32_t)((int32_t)hi[i] >> 31);
        const uint32_t t = (hi[i] ^ (s | 0x80000000u)) - 0x00100000u;  // monotone in the value; non-finite -> >= 0xFFE00000
        key[i] = (t | IDX) - (IDX - (uint32_t)i);                       // (t & ~IDX) | i
        const uint32_t z = t - kKeyNonFinite;
        const uint32_t u = z - Z_NONE;
        const uint32_t tagged_inc = (u < 2u) ? (u + 0x10100u) : 0x100u;
        census += (z < 0x00200000u) ? tagged_inc : 0u;
    }
    const int m = N - (int)((census >> 8) & 0xFFu);   // finite cells (cu:1105-1114)
    const int present = N - (int)(census & 0xFFu);    // len(values) at this node
    const int nn = N - (int)(census >> 16);           // non-None cells == `total` (cu:1100)
    if (nn == 0) {
        value = qnan;
        meta = pack_meta(0, 0, 0, present, 0);
        return;
    }
    if (nn == 1) {  // cu:1085-1086: the original object, whatever it is (rare: scan row memory for the untagged cell)
        int idx = 0;
        for (int i = 0; i < N; ++i) {
            const uint32_t h = lds_u32x2(row.addr(i)).y;
            if (h != kNoneHi && h != kAbsentHi) idx = i;
        }
        value = lds_f64(row.addr(idx));
        meta = pack_meta(idx, 1, 1, present, KC_FLAG_HAS_VALUE | KC_FLAG_SINGLE);
        return;
    }
    if (m == 0) {  // cu:1115-1116
        value = qnan;
        meta = pack_meta(0, 0, nn, present, KC_FLAG_NO_FINITE);
        return;
    }

    // D. sort keys; E. fetch the cells in key order
    sort_keys<N>(key);
    double xs[N];
#pragma unroll
    for (int k = 0; k < N; ++k) xs[k] = lds_f64(row.addr_mad(key[k] & IDX));

    // Keys drop low mantissa bits: values that differ only there may be swapped.  (NaN compares false; a -inf in
    // the non-finite tail can raise a false alarm, which only costs the repair call.)
    bool unsorted = false;
#pragma unroll
    for (int k = 1; k < N; ++k) unsorted |= xs[k] < xs[k - 1];
    // G. park the sorted values in row memory for the data-dependent ranges below
#pragma unroll
    for (int k = 0; k < N; ++k) sts_f64(row.addr(k), xs[k]);
    if (unsorted) {  // rare: insertion-sort the finite prefix in row memory, then reload
        repair_sorted_prefix<Row>(row, m);
#pragma unroll
        for (int k = 0; k < N; ++k) xs[k] = lds_f64(row.addr(k));
    }

    // F. cluster starts: bit k set <=> xs[k] opens a cluster (not close to xs[k-1]); cu:1130-1143.
    //    For a <= b:  |b-a| <= max(abs_eps, rel*max(|a|,|b|,1))
    //            <=>  (b-a) <= rel*b  or  (b-a) <= rel*(-a)  or  (b-a) <= max(abs_eps, rel)
    //    (max(|a|,|b|) = max(-a, b) for a <= b; fl(rel * .) is monotone for rel >= 0, so the product of the max is
    //    the max of the products.)  Pairs that touch the non-finite tail are masked off below.
    M starts = 1;
    {
        double p_prev = __dmul_rn(rel_eps, xs[0]);
#pragma unroll
        for (int k = 1; k < N; ++k) {
            const double p = __dmul_rn(rel_eps, xs[k]);
            const double d = __dadd_rn(xs[k], -xs[k - 1]);
            starts |= (M)far_bit(d, p, -p_prev, thr, 1u << (k & 31)) << (k & 32);
            p_prev = p;
        }
    }
    if (m < N) starts &= (M(1) << m) - 1;  // m >= 1 here

    // H. largest cluster
    int top = 0, n_top = 0, top_s = 0;
    {   // a cluster holding a strict majority of the finite values must contain the middle one: test that first
        const int c = m >> 1;
        const M below = starts & ((M(2) << c) - 1);          // starts at or below c (bit 0 is always set)
        const int s0 = (int)(sizeof(M) * 8 - 1) - clz_m(below);
        const M above = c + 1 < (int)(sizeof(M) * 8) ? (starts >> (c + 1)) : M(0);
        const int e0 = above ? c + ffs_m(above) : m;
        if (2 * (e0 - s0) > m) {
            top = e0 - s0;
            n_top = 1;
            top_s = s0;
        }
    }
    if (n_top == 0) {
        M sk = starts;
        while (sk) {
            const int s = ffs_m(sk) - 1;
            sk &= sk - 1;
            const int e = sk ? ffs_m(sk) - 1 : m;
            const int len = e - s;
            if (len > top) {
                top = len;
                n_top = 1;
                top_s = s;
            } else if (len == top) {
                ++n_top;
            }
        }
    }
    uint32_t flags = KC_FLAG_HAS_VALUE;
    int support = top;
    if (n_top == 1) {
        if constexpr (N <= 16 && std::is_same<Row, PlaneRow>::value)
            value = np_mean16(row, top_s, top);  // cu:1174-1178 / 1183-1187
        else
            value = np_mean(row, top_s, top);
    } else {
        const TieResult tr = numeric_tie<M, Row>(row, starts, m, top, rel_eps, abs_eps);
        value = tr.value;
        support = tr.support;
        flags |= KC_FLAG_TIE;
    }
    meta = pack_meta(0, support, nn, present, flags);
}

// ---------------------------------------------------------------- n = 2: the whole algorithm by cases
//
// Two cells leave a handful of outcomes (cu:1082-1219 restated for n = 2; oracle/consensus_oracle.c is the spec):
//   no non-None cell          -> no value                                   one non-None cell -> that cell (SINGLE)
//   two non-None, none finite -> NO_FINITE                                   one finite        -> 0.0 + v, support 1 of 2
//   two finite, close         -> ((-0.0 + lo) + hi + 0.0) / 2, support 2     two finite, far   -> tie of two singletons: the larger
//                                                                               |value| (the smaller on equal magnitudes), TIE
// The generic kernels pay ~470 instructions per group for their census / sort / queue machinery whatever n is (round 1: 0.21 of
// the HBM peak at n = 2); this is ~60.  A thread owns FOUR consecutive groups = 64 bytes of cells (four 16-byte loads, the next
// 64 bytes requested first) and writes its results as vectors.
__device__ __forceinline__ void numeric_pair(uint2 a, uint2 b, double rel_eps, double abs_eps, double &value, uint32_t &meta) {
    const bool a_abs = a.y == kAbsentHi, b_abs = b.y == kAbsentHi;
    const bool a_nn = !a_abs && a.y != kNoneHi, b_nn = !b_abs && b.y != kNoneHi;
    const bool a_fin = a_nn && (a.y & 0x7FF00000u) != 0x7FF00000u, b_fin = b_nn && (b.y & 0x7FF00000u) != 0x7FF00000u;
    const uint32_t present = (a_abs ? 0u : 1u) + (b_abs ? 0u : 1u), nn = (a_nn ? 1u : 0u) + (b_nn ? 1u : 0u);
    const double va = __hiloint2double((int)a.y, (int)a.x), vb = __hiloint2double((int)b.y, (int)b.x);
    const double qnan = __longlong_as_double(0x7FF8000000000000ll);
    if (nn == 0) {
        value = qnan;
        meta = pack_meta(0, 0, 0, present, 0);
    } else if (nn == 1) {  // the original object, untouched (cu:1085-1086)
        value = a_nn ? va : vb;
        meta = pack_meta(a_nn ? 0u : 1u, 1, 1, present, KC_FLAG_HAS_VALUE | KC_FLAG_SINGLE);
    } else if (!a_fin && !b_fin) {  // cu:1115-1116
        value = qnan;
        meta = pack_meta(0, 0, 2, present, KC_FLAG_NO_FINITE);
    } else if (a_fin != b_fin) {  // one finite value: its own cluster, np.mean of one element
        value = __dadd_rn(0.0, __dadd_rn(-0.0, a_fin ? va : vb));
        meta = pack_meta(0, 1, 2, present, KC_FLAG_HAS_VALUE);
    } else {
        const bool swap = va > vb;  // xs.sort(): ascending, equal elements keep their order
        const double lo = swap ? vb : va, hi = swap ? va : vb;
        if (is_close(lo, hi, rel_eps, abs_eps)) {
            value = __ddiv_rn(__dadd_rn(0.0, __dadd_rn(__dadd_rn(-0.0, lo), hi)), 2.0);
            meta = pack_meta(0, 2, 2, present, KC_FLAG_HAS_VALUE);
        } else {  // two singleton clusters tie: equal support and spread, the larger |center| wins, else the first (lower) one
            const double c_lo = __dadd_rn(0.0, __dadd_rn(-0.0, lo)), c_hi = __dadd_rn(0.0, __dadd_rn(-0.0, hi));
            value = fabs(c_hi) > fabs(c_lo) ? c_hi : c_lo;
            meta = pack_meta(0, 1, 2, present, KC_FLAG_HAS_VALUE | KC_FLAG_TIE);
        }
    }
}

__global__ void __launch_bounds__(256) numeric_pairs_kernel(const double *__restrict__ vals, int64_t n_units, double rel_eps, double abs_eps,
                                                            double *__restrict__ out_value, uint32_t *__restrict__ out_meta) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    prefetch_units<4>(vals, (int64_t)blockIdx.x * blockDim.x + threadIdx.x, n_units, stride, [&](int64_t u, const int4 (&cur)[4]) {
        double v[4];
        uint32_t m[4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
            numeric_pair(make_uint2((uint32_t)cur[q].x, (uint32_t)cur[q].y), make_uint2((uint32_t)cur[q].z, (uint32_t)cur[q].w), rel_eps, abs_eps,
                         v[q], m[q]);
        double *ov = out_value + u * 4;
        asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(ov), "d"(v[0]), "d"(v[1]) : "memory");
        asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(ov + 2), "d"(v[2]), "d"(v[3]) : "memory");
        asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(out_meta + u * 4), "r"(m[0]), "r"(m[1]), "r"(m[2]), "r"(m[3])
                     : "memory");
    });
}

// ---------------------------------------------------------------- n = 4: sort four, read the cluster pattern off three bits
//
// With at most four finite cells the clusters are the runs of the three "adjacent values are close" bits, and a tie between
// equally large clusters can only be all-singletons or two pairs — in both there is no strictly smaller cluster to lend
// support (cu:1189-1208 adds nothing), so the tie order (spread, then |center|, cu:1211) is all that is left.  ~150 instructions
// per group against ~470 for the generic fast kernel.  Two groups per thread.
__device__ __forceinline__ void cex(double &a, double &b) {  // compare-exchange, ascending; equal values keep their places
    const bool sw = a > b;
    const double lo = sw ? b : a, hi = sw ? a : b;
    a = lo;
    b = hi;
}

__device__ __forceinline__ void numeric_quad(const uint2 (&w)[4], double rel_eps, double abs_eps, double &value, uint32_t &meta) {
    const double pinf = __longlong_as_double(0x7FF0000000000000ll), qnan = __longlong_as_double(0x7FF8000000000000ll);
    uint32_t present = 0, nn = 0, m = 0, first_nn = 0;
    double x[4];
#pragma unroll
    for (int i = 3; i >= 0; --i) {  // descending, so that first_nn ends on the FIRST non-None cell
        const bool absent = w[i].y == kAbsentHi, none = w[i].y == kNoneHi, fin = (w[i].y & 0x7FF00000u) != 0x7FF00000u;
        present += absent ? 0u : 1u;
        const bool is_nn = !absent && !none;
        nn += is_nn ? 1u : 0u;
        first_nn = is_nn ? (uint32_t)i : first_nn;
        m += fin ? 1u : 0u;
        x[i] = fin ? __hiloint2double((int)w[i].y, (int)w[i].x) : pinf;  // non-finite cells sort behind every finite value
    }
    if (nn == 0) {
        value = qnan;
        meta = pack_meta(0, 0, 0, present, 0);
        return;
    }
    if (nn == 1) {  // the original object, untouched (cu:1085-1086)
        const uint2 c = first_nn == 0 ? w[0] : (first_nn == 1 ? w[1] : (first_nn == 2 ? w[2] : w[3]));
        value = __hiloint2double((int)c.y, (int)c.x);
        meta = pack_meta(first_nn, 1, 1, present, KC_FLAG_HAS_VALUE | KC_FLAG_SINGLE);
        return;
    }
    if (m == 0) {  // cu:1115-1116
        value = qnan;
        meta = pack_meta(0, 0, nn, present, KC_FLAG_NO_FINITE);
        return;
    }
    // xs.sort(): a stable 5-comparator network on (value, original place is irrelevant: equal doubles are interchangeable
    // in every sum below, and +0.0 / -0.0 only differ when ALL summands are zeros of one sign, which any order preserves)
    cex(x[0], x[1]);
    cex(x[2], x[3]);
    cex(x[0], x[2]);
    cex(x[1], x[3]);
    cex(x[1], x[2]);
    // runs of close neighbours among the m finite values (cu:1127-1144)
    const bool b0 = m > 1 && is_close(x[0], x[1], rel_eps, abs_eps);
    const bool b1 = m > 2 && is_close(x[1], x[2], rel_eps, abs_eps);
    const bool b2 = m > 3 && is_close(x[2], x[3], rel_eps, abs_eps);
    uint32_t best_len = 0, best_start = 0, n_top = 0, cur_len = 0, cur_start = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const bool in = (uint32_t)i < m;
        const bool joins = i > 0 && (i == 1 ? b0 : (i == 2 ? b1 : b2));
        cur_start = joins ? cur_start : (uint32_t)i;
        cur_len = joins ? cur_len + 1u : 1u;
        const bool ends = in && ((uint32_t)i + 1u == m || !(i == 0 ? b0 : (i == 1 ? b1 : b2)));
        if (ends) {
            if (cur_len > best_len) {
                best_len = cur_len;
                best_start = cur_start;
                n_top = 1;
            } else if (cur_len == best_len) {
                ++n_top;
            }
        }
    }
    // float(np.mean(x[s .. s+z))): -0.0 + x_s + ... left to right, + 0.0, / z
    auto mean_of = [&](uint32_t s, uint32_t z) -> double {
        double acc = -0.0;
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if ((uint32_t)i >= s && (uint32_t)i < s + z) acc = __dadd_rn(acc, x[i]);
        return __ddiv_rn(__dadd_rn(0.0, acc), (double)z);
    };
    if (n_top == 1) {  // cu:1171-1187
        value = mean_of(best_start, best_len);
        meta = pack_meta(0, best_len, nn, present, KC_FLAG_HAS_VALUE);
        return;
    }
    if (best_len == 1) {  // singletons: equal support and spread; the larger |center| wins, the first (lowest) one on equality
        double best = __dadd_rn(0.0, __dadd_rn(-0.0, x[0]));
#pragma unroll
        for (int i = 1; i < 4; ++i) {
            const double c = __dadd_rn(0.0, __dadd_rn(-0.0, x[i]));
            if ((uint32_t)i < m && fabs(c) > fabs(best)) best = c;
        }
        value = best;
        meta = pack_meta(0, 1, nn, present, KC_FLAG_HAS_VALUE | KC_FLAG_TIE);
        return;
    }
    // two pairs (x0, x1) and (x2, x3): smaller np.std first, then the larger |median| (= |mean| of the pair)
    auto pair_stats = [&](double a, double b, double &mean, double &sd) {
        mean = __ddiv_rn(__dadd_rn(0.0, __dadd_rn(__dadd_rn(-0.0, a), b)), 2.0);
        const double ta = __dadd_rn(a, -mean), tb = __dadd_rn(b, -mean);
        const double ss = __dadd_rn(0.0, __dadd_rn(__dadd_rn(-0.0, __dmul_rn(ta, ta)), __dmul_rn(tb, tb)));
        sd = __dsqrt_rn(__ddiv_rn(ss, 2.0));
    };
    double ma, sa, mb, sb;
    pair_stats(x[0], x[1], ma, sa);
    pair_stats(x[2], x[3], mb, sb);
    const bool second = sb < sa || (sb == sa && fabs(mb) > fabs(ma));
    value = second ? mb : ma;
    meta = pack_meta(0, 2, nn, present, KC_FLAG_HAS_VALUE | KC_FLAG_TIE);
}

__global__ void __launch_bounds__(256) numeric_quads_kernel(const double *__restrict__ vals, int64_t n_units, double rel_eps, double abs_eps,
                                                            double *__restrict__ out_value, uint32_t *__restrict__ out_meta) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    prefetch_units<4>(vals, (int64_t)blockIdx.x * blockDim.x + threadIdx.x, n_units, stride, [&](int64_t u, const int4 (&cur)[4]) {
        double v[2];
        uint32_t m[2];
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            const uint2 w[4] = {make_uint2((uint32_t)cur[2 * g].x, (uint32_t)cur[2 * g].y), make_uint2((uint32_t)cur[2 * g].z, (uint32_t)cur[2 * g].w),
                                make_uint2((uint32_t)cur[2 * g + 1].x, (uint32_t)cur[2 * g + 1].y),
                                make_uint2((uint32_t)cur[2 * g + 1].z, (uint32_t)cur[2 * g + 1].w)};
            numeric_quad(w, rel_eps, abs_eps, v[g], m[g]);
        }
        asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(out_value + u * 2), "d"(v[0]), "d"(v[1]) : "memory");
        asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(out_meta + u * 2), "r"(m[0]), "r"(m[1]) : "memory");
    });
}

// (The same shape for n = 8 — a 19-comparator network on the doubles, seven closeness bits, numeric_tie for the rare ties — was
// built, is bit-exact, and is slower than the adder-tree fast path.  Sorting and chaining eight doubles in
// FP64 compares costs more than proving a majority on 32-bit words; removed.)

// ---------------------------------------------------------------- direct front-end (any n <= NP)

// dynamic shared memory of the direct kernels (numeric_direct_kernel, numeric_direct_fast_kernel): the [cell][thread] plane
template <int NP, int T>
constexpr size_t numeric_direct_smem() {
    return (size_t)NP * T * 8;
}

template <int NP, int T, bool PREFETCH>
__global__ void __launch_bounds__(T) numeric_direct_kernel(const double *__restrict__ vals, int64_t n_groups, int n,
                                                           double rel_eps, double abs_eps, double *__restrict__ out_value,
                                                           uint32_t *__restrict__ out_meta, const __grid_constant__ OutRoute mc) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const PlaneRow row{smem_u32(smem_raw) + threadIdx.x * 8u, T * 8u};
    const double thr = abs_eps > rel_eps ? abs_eps : rel_eps;
    const int64_t stride = (int64_t)gridDim.x * T;
    int64_t g = (int64_t)blockIdx.x * T + threadIdx.x;
    int4 cur[NP / 2];
    if (PREFETCH && g < n_groups) load_cells(vals + g * NP, cur);  // PREFETCH requires n == NP
    for (; g < n_groups; g += stride) {
        const double *p = vals + g * n;
        uint32_t hi[NP];
        int4 nxt[NP / 2];
        if (PREFETCH || n == NP) {
            if constexpr (PREFETCH) {
                if (g + stride < n_groups) load_cells(vals + (g + stride) * NP, nxt);  // request the next row before working on this one
            } else {
                load_cells(p, cur);
            }
#pragma unroll
            for (int q = 0; q < NP / 2; ++q) load_pair(cur[q], q, hi, row);
        } else {
#pragma unroll
            for (int i = 0; i < NP; ++i) {
                const double v = (i < n) ? __ldg(p + i) : __longlong_as_double((long long)KC_F64_ABSENT_BITS);
                hi[i] = (uint32_t)__double2hiint(v);
                sts_f64(row.addr(i), v);
            }
        }
        double v;
        uint32_t m;
        numeric_core<NP, PlaneRow>(hi, row, rel_eps, abs_eps, thr, v, m);
        store_out_f64(out_value + g, v, mc);
        store_out_u32(out_meta + g, m, mc);
        if constexpr (PREFETCH) {
#pragma unroll
            for (int q = 0; q < NP / 2; ++q) cur[q] = nxt[q];
        }
    }
}

// ---------------------------------------------------------------- TMA front-end (n in {4,8,16,32,64})

// Warp-private pipelines exactly as vote_tma_kernel; rows are n*8 bytes (box rows are at most 128 B wide, the
// widest TMA swizzle span, so wider rows are several box rows).  The swizzled tile is read ONCE with static,
// conflict-free LDS.128 and copied to a [cell][thread] plane: the data-dependent accesses of the core would
// bank-conflict on a row-per-thread layout, while in the plane the bank depends on the thread only.  The stage
// is handed back to the TMA unit right after that copy.

// dynamic shared memory of the TMA kernels (numeric_tma_kernel, numeric_tma_fast_kernel): the rings, then the plane
template <int N, int WARPS, int STAGES>
constexpr size_t numeric_tma_smem() {
    return WarpTiles<N * 8, WARPS, STAGES>::RING_BYTES + numeric_direct_smem<N, WARPS * 32>();
}

// ---------------------------------------------------------------- K2 fast path: a strict majority of identical cells
//
// Candidates of one field mostly agree bit for bit.  If one value v fills a strict majority of the m finite cells, its
// cluster is the unique largest one whatever the rest looks like (cu:1145-1187), and if no other finite cell is close
// to v the cluster is exactly the c copies of v: value = np.mean([v]*c), support = c — no sort, no closeness chain.
// With one or two cells chained to v the cluster is still known: those extras, then the copies, in sorted order.
//   1. guess v as the bitwise "at least half" vote over the cells (carry-save adder tree, kc_csa.cuh);
//   2. verify exactly: c = cells bit-identical to v, 2c > m;
//   3. the nearest finite cells below and above v are found on the HIGH words only (two unsigned min/max scans; only
//      groups without negative cells are taken, so raw high words are ordered like the values); each stands for every
//      double sharing that high word.  They are certified far from v with
//      fl() monotonicity alone: |v - x| >= fl(v - x_nearest_possible) and tol(x, v) <= max(abs, fl(rel * max(|x|_max,
//      |v|, 1))) for rel >= 0 (the launcher rejects rel < 0).  A neighbour that cannot be certified so is completed from
//      the one cell with its high word, tested exactly (far_bit, as numeric_core's chain) and, if close, taken as an
//      extra; the walk goes on from it, for at most two extras in all;
//   4. the cell census comes from the same adder tree (bit 31 of x = hi + 2^20 counts the non-finite cells) plus one
//      min scan that proves every non-finite cell is a None / absent tag;
//   5. anything else — no majority, a third extra, a neighbour sharing its high word with another cell, a cell sharing
//      v's high word, a negative cell, an inf or an untagged NaN, a single non-None cell — is NOT decided here: the caller
//      parks the group for numeric_core
//      (exact, general).
// numeric_fast_decide() returns true when the group is decided; numeric_fast_finish() then produces (value, meta).
// n += (x == key), as a predicated add (the compiler prefers select + add)
__device__ __forceinline__ void count_equal(uint32_t x, uint32_t key, uint32_t &n) {
    asm("{\n\t.reg .pred p;\n\t"
        "setp.eq.u32 p, %1, %2;\n\t"
        "@p add.u32 %0, %0, 1;\n\t}"
        : "+r"(n)
        : "r"(x), "r"(key));
}

// a cell with v's high word: count it, and collect any difference of its low word
__device__ __forceinline__ void match_cell(uint32_t h, uint32_t l, uint32_t hv, uint32_t lv, uint32_t &c, uint32_t &bad) {
    asm("{\n\t.reg .pred p;\n\t"
        "setp.eq.u32 p, %2, %4;\n\t"
        "@p add.u32 %0, %0, 1;\n\t"
        "@p lop3.b32 %1, %1, %3, %5, 0xF6;\n\t}"  // bad | (l ^ lv)
        : "+r"(c), "+r"(bad)
        : "r"(h), "r"(l), "r"(hv), "r"(lv));
}

// Callers pass x = hi + 2^20 (kFastBias) for every cell and top = the largest raw high word (unsigned).
constexpr uint32_t kFastBias = 0x00100000u;

// the row loader's load_pair for numeric_fast_decide: cells 2q and 2q+1 into x[] and lo[], their high words into top
template <int N>
__device__ __forceinline__ void fast_pair(const int4 &c, int q, uint32_t (&x)[N], uint32_t (&lo)[N], uint32_t &top) {
    lo[2 * q + 0] = (uint32_t)c.x;
    x[2 * q + 0] = (uint32_t)c.y + kFastBias;
    lo[2 * q + 1] = (uint32_t)c.z;
    x[2 * q + 1] = (uint32_t)c.w + kFastBias;
    top = max(top, max((uint32_t)c.y, (uint32_t)c.w));
}

struct FastDecision {
    double v;       // the majority value
    double e0, e1;  // the extras chained to v, the last found first (the walk goes down from v, then up)
    // the result word with v's copies as the support, and in the first-seen index bits (0 in the result) the number of
    // extras below v (bits 0-1) and above it (bits 2-3): one register while the cells are still live
    uint32_t word;
};

// The walk to extras pays off from n = 16 (the share of groups with a close neighbour grows with n); at n = 8 it measured
// slower on H100 than deferring those groups, so there every group with a close neighbour is deferred, and the finish
// sums the copies of v alone.
template <int N>
constexpr bool kWalkExtras = N >= 16;

// Every double with the high word h lies beyond reach of f: h below f's high word (below) or above it.  fl(rel * .) is
// monotone, so it is enough that the least possible distance exceeds thr = max(abs, rel) and rel * the largest magnitude.
__device__ __forceinline__ bool certainly_far(double f, uint32_t h, bool below, double rel_eps, double thr) {
    const double d = below ? __dadd_rn(f, -__hiloint2double((int)h, -1)) : __dadd_rn(__hiloint2double((int)h, 0), -f);
    const double mag = below ? f : __hiloint2double((int)h, -1);
    return d > thr && d > __dmul_rn(rel_eps, mag);
}

// Phase 1: decide.  True <=> the group's result is the mean of v's copies and the extras in `out`; the cells are not needed
// afterwards.
template <int N>
__device__ __forceinline__ bool numeric_fast_decide(const uint32_t (&x)[N], const uint32_t (&lo)[N], uint32_t top, double rel_eps,
                                                    double thr, FastDecision &out) {
    // Only groups whose largest high word (unsigned) is at most the absent tag are decided here: no negative cell (-0.0
    // included), no NaN payload above the tags; raw high words of non-negative doubles are ordered like the values.
    // x = hi + 2^20 then has bit 31 set <=> the cell is not finite (exponent all ones).
    constexpr uint32_t X_NONE = kNoneHi + kFastBias, X_ABSENT = kAbsentHi + kFastBias;
    constexpr int PLANES = 32 - __builtin_clz((unsigned)N);  // weights 1 .. N
    // per bit position, how many cells have the bit set: the two top planes give the "at least half" guess of v's
    // high word, bit 31 of all planes the number of non-finite cells
    uint32_t plane[PLANES];
    bit_counts(x, plane);
    const uint32_t xv = plane[PLANES - 1] | plane[PLANES - 2], lv = at_least_half(lo);
    uint32_t nonfinite = 0;
#pragma unroll
    for (int k = 0; k < PLANES; ++k) nonfinite += (plane[k] >> 31) << k;
    // d = x - xv as a signed number: < 0 below v, > 0 above.  Unsigned max of d is the nearest cell below (if any is
    // below), unsigned min of d - 1 the nearest above.
    // low_nf: the smallest non-finite x, as an offset from 2^31 (finite cells wrap to >= 2^31 and never win the min)
    uint32_t c = 0, bad = 0, below = 0, above = 0xFFFFFFFFu, low_nf = 0xFFFFFFFFu, absent = 0;
    const uint32_t neg_xv = 0u - xv, neg_xv1 = ~xv;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        below = max(below, x[i] + neg_xv);
        above = min(above, x[i] + neg_xv1);
        low_nf = min(low_nf, x[i] + 0x80000000u);
        match_cell(x[i], lo[i], xv, lv, c, bad);
    }
    if (top == kAbsentHi) {  // ragged candidates (rare): count the absent cells
#pragma unroll
        for (int i = 0; i < N; ++i) count_equal(x[i], X_ABSENT, absent);
    }
    // With no non-finite cell below the None tag (inf, a plain NaN: decided by the general path) and none above the absent
    // tag (`top`), every non-finite cell is None or absent.
    const uint32_t tagged = nonfinite;
    // a negative cell or an odd NaN / the guess is not a finite value / cells share v's high word only / no strict
    // majority of the finite cells / a single non-None cell / an untagged non-finite cell
    if (top > kAbsentHi || (xv & 0x80000000u) != 0 || bad != 0 || 2 * c + nonfinite <= (uint32_t)N || tagged > (uint32_t)(N - 2) ||
        (nonfinite != 0 && low_nf < X_NONE - 0x80000000u))
        return false;
    const uint32_t hv = xv - kFastBias;
    const double v = __hiloint2double((int)hv, (int)lv);
    // Neighbours: every double with the high word hb is <= (hb, ~0) < v, every one with ha is in [(ha, 0), (ha, ~0)].
    // close(a, b) <=> |a-b| <= max(abs, rel*max(|a|,|b|,1)) = max(thr, fl(rel*max(|a|,|b|))) with thr = max(abs, rel),
    // because fl(rel * .) is monotone; so "certainly far" <=> d > thr and d > fl(rel * upper bound of the magnitudes).
    const uint32_t hb = hv + below, ha = hv + above + 1u;
    const bool has_b = below >= 0x80000000u, has_a = above < 0x7FFFFFFFu && ha < 0x7FF00000u;
    const bool need_b = has_b && !certainly_far(v, hb, true, rel_eps, thr);
    const bool need_a = has_a && !certainly_far(v, ha, false, rel_eps, thr);
    out.v = v;
    out.word = (c << 6) + (((uint32_t)N - tagged) << 13) + (((uint32_t)N - absent) << 20) + ((uint32_t)KC_FLAG_HAS_VALUE << 27);
    out.e0 = out.e1 = v;
    // A neighbour within possible reach: walk outwards from v, one cell per step, below v first.  A step needs the
    // neighbour's high word to be unique among the cells (that cell's low word completes it), tests it exactly as
    // numeric_core's chain does, and if it is close takes it as an extra and certifies the next cell beyond it far.  At
    // most two extras; anything else is left to the general path.
    // xn: the neighbour under test (biased high word, below xv while walking down), xa: where the upward walk starts
    // (0: nowhere, and xn = 0 ends the walk)
    if constexpr (!kWalkExtras<N>) {
        if (need_b || need_a) return false;
    }
    uint32_t xn = need_b ? hb + kFastBias : 0u, xa = need_a ? ha + kFastBias : 0u;
    if (xn == 0u) {
        xn = xa;
        xa = 0u;
    }
    while (xn != 0u) {
        const uint32_t nb = out.word & 3u, na = (out.word >> 2) & 3u;
        if (nb + na == 2u) return false;
        const bool down = xn < xv;
        // beyond: as `below` / `above` from xn, mirrored for the upward walk (>= 2^31 <=> a cell lies beyond xn)
        const uint32_t sm = down ? 0u : 0xFFFFFFFFu, neg = 0u - (xn ^ sm);
        uint32_t cnt = 0, ln = 0, beyond = 0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            beyond = max(beyond, (x[i] ^ sm) + neg);
            asm("{\n\t.reg .pred p;\n\t"
                "setp.eq.u32 p, %2, %4;\n\t"
                "@p add.u32 %0, %0, 1;\n\t"
                "@p mov.b32 %1, %3;\n\t}"
                : "+r"(cnt), "+r"(ln)
                : "r"(x[i]), "r"(lo[i]), "r"(xn));
        }
        if (cnt != 1u) return false;
        const double e = __hiloint2double((int)(xn - kFastBias), (int)ln);
        const double f = (down ? nb : na) ? out.e0 : v;  // the cluster's outermost value on this side so far
        const double a = down ? e : f, b = down ? f : e;
        const bool close = far_bit(__dadd_rn(b, -a), __dmul_rn(rel_eps, b), -__dmul_rn(rel_eps, a), thr, 1u) == 0u;
        bool side_done = !close;
        if (close) {
            out.e1 = out.e0;
            out.e0 = e;
            out.word += down ? 1u : 4u;
            const uint32_t hn = (down ? xn + beyond : xn - beyond) - kFastBias;
            const bool exists = beyond >= 0x80000000u && (down || hn < 0x7FF00000u);
            side_done = !exists || certainly_far(e, hn, down, rel_eps, thr);
            xn = hn + kFastBias;
        }
        if (side_done) {
            xn = xa;
            xa = 0u;
        }
    }
    return true;
}

// Phase 2: the value and the result word of a decided group.
template <int N>
__device__ __forceinline__ void numeric_fast_finish(const FastDecision &d, double &value, uint32_t &meta) {
    const double v = d.v;
    const uint32_t c = (d.word >> 6) & 127u;
    if constexpr (!kWalkExtras<N>) {
        // c copies of v alone: for c >= 8 the eight accumulators are identical (r = the sequential sum of c/8 copies) and
        // their pairwise sum is 8r exactly; then the c%8 stragglers one by one.
        double res = -0.0;  // -0.0 + v == v
        if (c >= 8) {
            double r = v;
#pragma unroll
            for (int k = 2; k <= N / 8; ++k)
                if ((int)(c >> 3) >= k) r = __dadd_rn(r, v);
            res = __dmul_rn(r, 8.0);
        }
#pragma unroll
        for (int k = 1; k <= 7; ++k)
            if ((int)(c & 7u) >= k) res = __dadd_rn(res, v);
        value = __ddiv_rn(__dadd_rn(0.0, res), (double)c);
        meta = d.word;
        return;
    }
    const uint32_t nb = d.word & 3u, na = (d.word >> 2) & 3u;
    const uint32_t z = c + nb + na, q = z >> 3, t = z & 7u;
    const double f0 = nb == 0u ? v : (na == 0u ? d.e0 : d.e1), f1 = nb == 2u ? d.e1 : v;  // first two in sorted order
    const double l2 = na == 2u ? d.e1 : v, l1 = na == 0u ? v : d.e0;                       // last two
    // np.mean of the sorted cluster [f0 f1 | v ... v | l2 l1] (nb extras first, na last) in numpy's summation order.
    // z >= 8: accumulator j sums the positions = j (mod 8) below z - t.  Extras below v can only open accumulators 0 and
    // 1; extras above v can only close accumulators 6 and 7 (t = 0: both, t = 1: the one before the last) or sit in the
    // tail.  So r2..r5 are the plain sum of q copies, and each other accumulator is one sequential sum with its extra.
    double r0 = f0, r1 = f1, rp = -0.0;  // rp: q - 1 copies (-0.0 + x == x)
#pragma unroll
    for (int k = 2; k <= N / 8; ++k)
        if ((int)q >= k) {
            r0 = __dadd_rn(r0, v);
            r1 = __dadd_rn(r1, v);
            rp = __dadd_rn(rp, v);
        }
    const double r6 = __dadd_rn(rp, t == 0u ? l2 : v), r7 = __dadd_rn(rp, t == 0u ? l1 : (t == 1u ? l2 : v));
    const double r2 = __dadd_rn(rp, v), s23 = __dadd_rn(r2, r2);
    const double tree = __dadd_rn(__dadd_rn(__dadd_rn(r0, r1), s23), __dadd_rn(s23, __dadd_rn(r6, r7)));
    // then left to right: z < 8 the whole cluster from -0.0, otherwise the tail (copies of v, then the extras above in it)
    const bool small = z < 8u;
    const uint32_t sb = small ? nb : 0u, sa = small ? na : min(na, t), sv = small ? c : t - sa;
    double res = small ? -0.0 : tree;
    if (sb >= 1u) res = __dadd_rn(res, f0);
    if (sb >= 2u) res = __dadd_rn(res, f1);
#pragma unroll
    for (int k = 1; k <= 7; ++k)
        if ((int)sv >= k) res = __dadd_rn(res, v);
    if (sa >= 2u) res = __dadd_rn(res, l2);
    if (sa >= 1u) res = __dadd_rn(res, l1);
    value = __ddiv_rn(__dadd_rn(0.0, res), (double)z);
    meta = (d.word & ~15u) + ((nb + na) << 6);
}

// ---------------------------------------------------------------- the fast kernels' deferral queue
//
// Cells stay in registers for the fast path; a group it does not decide parks its cells in one of the warp's 32 plane rows
// (slot s = the row of lane s) and its index in the warp's 64 `slot` entries.  When 32 wait, the warp runs numeric_core on
// them with every lane busy: the general path costs its instructions only for the groups that need it.  Groups parked
// past the 32nd keep only their index; when they move down, their cells are fetched again from `rows` (a few groups at
// most).  Whole warps call put() together, once per step (so that the count stays warp-uniform), and finish() at the end.
// A kernel passes its plane (the first 8-byte cell of thread 0), the warp's first thread, and the warp's row of slots.
// The kernels call numeric_fast_decide themselves: called inside put(), it compiles the TMA kernels to other code.
template <int N, int T, typename Idx>
struct DeferQueue {
    int count = 0;  // warp-uniform; the first member, since the member order shows in the fast kernels' register allocation
    Idx *slot;
    const double *rows;  // group g's cells at rows + g * N
    double *out_value;
    uint32_t *out_meta;
    double rel_eps, abs_eps, thr;
    PlaneRow row;  // this lane's
    uint32_t warp_plane, lane;

    __device__ __forceinline__ DeferQueue(Idx *slot_, uint32_t plane, uint32_t warp_thread0, uint32_t lane_, const double *rows_,
                                          double rel_eps_, double abs_eps_, double *out_value_, uint32_t *out_meta_)
        : slot(slot_), rows(rows_), out_value(out_value_), out_meta(out_meta_), rel_eps(rel_eps_), abs_eps(abs_eps_),
          thr(abs_eps_ > rel_eps_ ? abs_eps_ : rel_eps_), row{plane + threadIdx.x * 8u, T * 8u}, warp_plane(plane + warp_thread0 * 8u),
          lane(lane_) {}

    // the first `n` parked groups through the general path, one per lane
    __device__ __forceinline__ void drain(int n) {
        if ((int)lane < n) {
            const Idx g = slot[lane];
            uint32_t hi[N];
            plane_hi(row, hi);
            double v;
            uint32_t m;
            numeric_core<N, PlaneRow>(hi, row, rel_eps, abs_eps, thr, v, m);
            store_local_f64(out_value + g, v);
            store_local_u32(out_meta + g, m);
        }
        __syncwarp();
    }

    // group g of this lane (g >= n_groups: none), cells as fast_pair loads them: stored if the fast path decided it, else parked
    __device__ __forceinline__ void put(Idx g, Idx n_groups, const uint32_t (&x)[N], const uint32_t (&lo)[N], bool decided,
                                        const FastDecision &fd) {
        const bool defer = !decided && g < n_groups;
        const uint32_t dm = __ballot_sync(0xFFFFFFFFu, defer);
        if (defer) {  // park the cells in a free plane row; past the 32nd only the index is kept (re-read below)
            const uint32_t s = (uint32_t)count + (uint32_t)__popc(dm & ((1u << lane) - 1u));
            slot[s] = g;
            if (s < 32u) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    sts_f64(warp_plane + s * 8u + (uint32_t)i * (T * 8u), __hiloint2double((int)(x[i] - kFastBias), (int)lo[i]));
            }
        }
        count += __popc(dm);
        if (decided && g < n_groups) {
            double v;
            uint32_t m;
            numeric_fast_finish<N>(fd, v, m);
            store_local_f64(out_value + g, v);
            store_local_u32(out_meta + g, m);
        }
        __syncwarp();
        if (count >= 32) {  // nothing of this step is live in registers any more
            drain(32);
            count -= 32;
            const Idx moved = ((int)lane < count) ? slot[32 + lane] : Idx(0);
            __syncwarp();
            if ((int)lane < count) {  // the overflow: fetch its cells again
                slot[lane] = moved;
                const int4 *p4 = reinterpret_cast<const int4 *>(rows + (size_t)moved * N);
#pragma unroll
                for (int q = 0; q < N / 2; ++q) put_pair(row, q, ldg_nc_v4(p4 + q));
            }
            __syncwarp();
        }
    }

    __device__ __forceinline__ void finish() {
        if (count > 0) drain(count);
    }
};

// Register-prefetch front-end (n == NP, small rows) with the fast path.
template <int NP, int T>
__global__ void __launch_bounds__(T) numeric_direct_fast_kernel(const double *__restrict__ vals, int64_t n_groups, double rel_eps,
                                                                double abs_eps, double *__restrict__ out_value,
                                                                uint32_t *__restrict__ out_meta, const __grid_constant__ OutRoute /* local only: see the launcher */) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ int64_t defer_q[T / 32][64];
    const uint32_t lane = threadIdx.x & 31;
    DeferQueue<NP, T, int64_t> queue(defer_q[threadIdx.x >> 5], smem_u32(smem_raw), threadIdx.x & ~31u, lane, vals, rel_eps, abs_eps, out_value,
                                     out_meta);
    const int64_t stride = (int64_t)gridDim.x * T;
    const int64_t g0 = (int64_t)blockIdx.x * T + threadIdx.x;
    int4 cur[NP / 2];
    if (g0 < n_groups) load_cells(vals + g0 * NP, cur);
    // whole warps iterate together (the tail lanes idle) so that the queue bookkeeping stays warp-uniform
    for (int64_t gw = g0 - lane; gw < n_groups; gw += stride) {
        const int64_t g = gw + lane;
        int4 nxt[NP / 2];
        if (g + stride < n_groups) load_cells(vals + (g + stride) * NP, nxt);  // request the next row before working on this one
        uint32_t x[NP], lo[NP], top = 0;
#pragma unroll
        for (int q = 0; q < NP / 2; ++q) fast_pair(cur[q], q, x, lo, top);
        FastDecision fd;
        const bool decided = numeric_fast_decide<NP>(x, lo, top, rel_eps, queue.thr, fd);
        queue.put(g, n_groups, x, lo, decided, fd);
#pragma unroll
        for (int q = 0; q < NP / 2; ++q) cur[q] = nxt[q];
    }
    queue.finish();
}

// The TMA pipeline of numeric_tma_kernel with the fast path in front; nothing is read twice but the queue's overflow.
template <int N, int WARPS, int STAGES, int MIN_CTAS>
__global__ void __launch_bounds__(WARPS * 32, MIN_CTAS) numeric_tma_fast_kernel(const __grid_constant__ CUtensorMap tmap,
                                                                      const double *__restrict__ in, uint32_t n_groups,
                                                                      double rel_eps, double abs_eps,
                                                                      double *__restrict__ out_value,
                                                                      uint32_t *__restrict__ out_meta) {
    constexpr int T = WARPS * 32;
    WarpTiles<N * 8, WARPS, STAGES> tiles(&tmap, n_groups);
    __shared__ uint32_t defer_q[WARPS][64];
    DeferQueue<N, T, uint32_t> queue(defer_q[tiles.warp], tiles.end(), tiles.warp * 32u, tiles.lane, in, rel_eps, abs_eps, out_value, out_meta);
    tiles.start(L2Policy::evict_normal);

    for (; tiles.t < tiles.n_tiles; tiles.next()) {
        const uint32_t tile = tiles.wait();
        uint32_t x[N], lo[N], touch = 0, top = 0;
#pragma unroll
        for (int q = 0; q < N / 2; ++q) {
            const int4 c = lds_v4(tile + tiles.at(q * 16));
            fast_pair(c, q, x, lo, top);
            touch |= (uint32_t)c.w;  // one word of every LDS.128 is enough to depend on all of them
        }
        tiles.release(touch);
        const uint32_t g = tiles.t * 32 + tiles.lane;
        FastDecision fd;
        const bool decided = numeric_fast_decide<N>(x, lo, top, rel_eps, queue.thr, fd);
        queue.put(g, n_groups, x, lo, decided, fd);
    }
    queue.finish();
}

template <int N, int WARPS, int STAGES, int MIN_CTAS>
__global__ void __launch_bounds__(WARPS * 32, MIN_CTAS) numeric_tma_kernel(const __grid_constant__ CUtensorMap tmap,
                                                                 uint32_t n_groups, double rel_eps, double abs_eps,
                                                                 double *__restrict__ out_value,
                                                                 uint32_t *__restrict__ out_meta, const __grid_constant__ OutRoute mc) {
    constexpr int T = WARPS * 32;
    WarpTiles<N * 8, WARPS, STAGES> tiles(&tmap, n_groups);
    const PlaneRow row{tiles.end() + threadIdx.x * 8u, T * 8u};
    const double thr = abs_eps > rel_eps ? abs_eps : rel_eps;
    tiles.start(L2Policy::evict_normal);

    for (; tiles.t < tiles.n_tiles; tiles.next()) {
        const uint32_t tile = tiles.wait();
        uint32_t hi[N];
        uint32_t touch = 0;
#pragma unroll
        for (int q = 0; q < N / 2; ++q) {
            const int4 c = lds_v4(tile + tiles.at(q * 16));
            load_pair(c, q, hi, row);
            touch |= (uint32_t)c.w;  // one word of every LDS.128 is enough to depend on all of them
        }
        tiles.release(touch);
        const uint32_t g = tiles.t * 32 + tiles.lane;
        if (g < n_groups) {
            double v;
            uint32_t m;
            numeric_core<N, PlaneRow>(hi, row, rel_eps, abs_eps, thr, v, m);
            store_out_f64(out_value + g, v, mc);
            store_out_u32(out_meta + g, m, mc);
        }
    }
}

}  // namespace kc
