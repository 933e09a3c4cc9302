// kc_vote.cuh — K1: vote consensus (mode with first-seen ties) over dictionary-coded groups.
//
// Replaces voting_consensus (reference consensus_utils.py:936-982) on pre-sanitised input.
// One thread owns one group (the n candidate cells of one field of one record) in registers.
// HBM-bound streaming op: 4n bytes in, 8 bytes out per group, O(1) integer ops per byte, no reuse,
// no tensor cores.  Two front-ends feed the same register core:
//   * vote_tma_kernel    — n in {8,16,32,64}: every WARP runs its own TMA pipeline (WarpTiles, kc_common.cuh);
//                          no block-wide barrier anywhere.
//   * vote_direct_kernel — any n <= 64 (and n <= 4 where a thread's cells are one coalesced vector load), on int32 or
//                          int8 cells.
#pragma once

#include "kc_common.cuh"

namespace kc {

template <int N>
struct MaskOf {
    using type = uint32_t;
};
template <>
struct MaskOf<64> {
    using type = uint64_t;
};
__device__ __forceinline__ int popc_m(uint32_t m) { return __popc(m); }
__device__ __forceinline__ int popc_m(uint64_t m) { return __popcll(m); }
__device__ __forceinline__ int ffs_mask(uint32_t m) { return __ffs((int)m); }
__device__ __forceinline__ int ffs_mask(uint64_t m) { return __ffsll((long long)m); }

// bitwise helpers, one LOP3 each
__device__ __forceinline__ uint32_t lop3_maj(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
__device__ __forceinline__ uint32_t lop3_xor3(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
// bitwise majority of five = (carry & (sum|d|e)) | (sum&d&e) with (sum, carry) the full adder of a,b,c
__device__ __forceinline__ uint32_t maj5(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e) {
    const uint32_t s = lop3_xor3(a, b, c), cy = lop3_maj(a, b, c);
    return (cy & (s | d | e)) | (s & d & e);
}

// A cheap GUESS of the mode: bitwise majority over (up to) 27 cells.  Wrong guesses cost time, never
// correctness.  At p_agree = 0.8 / n = 16 it is the strict-majority value for 99.6 % of the groups.
template <int N>
__device__ __forceinline__ int32_t guess_mode(const int32_t (&x)[N]) {
    auto u = [&](int i) { return (uint32_t)x[i]; };
    if constexpr (N >= 27) {
        uint32_t t[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) t[i] = lop3_maj(u(3 * i), u(3 * i + 1), u(3 * i + 2));
        return (int32_t)lop3_maj(lop3_maj(t[0], t[1], t[2]), lop3_maj(t[3], t[4], t[5]), lop3_maj(t[6], t[7], t[8]));
    } else if constexpr (N >= 15) {
        return (int32_t)maj5(lop3_maj(u(0), u(1), u(2)), lop3_maj(u(3), u(4), u(5)), lop3_maj(u(6), u(7), u(8)),
                             lop3_maj(u(9), u(10), u(11)), lop3_maj(u(12), u(13), u(14)));
    } else if constexpr (N >= 8) {
        return (int32_t)lop3_maj(lop3_maj(u(0), u(1), u(2)), lop3_maj(u(3), u(4), u(5)), lop3_maj(u(6), u(7), u(0)));
    } else if constexpr (N >= 3) {
        return (int32_t)lop3_maj(u(0), u(1), u(2));
    } else {
        return x[0];
    }
}

// Exact first-seen-order scan (the general case).  x[i] >= 0 votes, x[i] < 0 does not.  Classes are visited
// in the order of their first cell and a later class must be STRICTLY larger to win, which is
// Counter.most_common(1) (cu:958,969).  The scan stops once the unvisited cells cannot reach the best count.
template <int N, typename M>
__device__ __forceinline__ uint32_t vote_scan(const int32_t (&x)[N], int present, int32_t &win_code) {
    M live = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) live |= (x[i] >= 0) ? (M(1) << i) : M(0);
    const int voters = popc_m(live);
    int best_cnt = 0, best_idx = 0;
    int32_t best_code = KC_CODE_NONE;
    bool tie = false;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if ((live >> i) & 1) {
            const int32_t c = x[i];
            M eq = 0;
#pragma unroll
            for (int j = i; j < N; ++j) eq |= (x[j] == c) ? (M(1) << j) : M(0);
            const int cnt = popc_m(eq);
            if (cnt > best_cnt) {
                best_cnt = cnt;
                best_idx = i;
                best_code = c;
                tie = false;
            } else if (cnt == best_cnt) {
                tie = true;
            }
            live &= ~eq;
            if (popc_m(live) < best_cnt) live = 0;  // nothing left can win or tie
        }
    }
    win_code = best_code;
    return pack_meta(best_idx, best_cnt, voters, present,
                     best_cnt > 0 ? (KC_FLAG_HAS_VALUE | (tie ? KC_FLAG_TIE : 0u)) : 0u);
}

// Mode of the voting cells of one group.  raw[i]: code >= 0, KC_CODE_NONE (-1) or absent (< -1).
// none_code >= 0 makes None cells vote as that code (bool fields: None -> False, cu:956).
//
// Fast path (no absent cell): None cells of fields where None votes are rewritten branch-free
// (x ^ (sign & ~none_code)); a bitwise-majority guess is counted with ONE equality pass; if it holds a strict
// majority of the voting cells it is the unique mode (no tie is possible) and its first cell is the first-seen
// original (cu:971).  Everything else falls through to the exact scan.
template <int N>
__device__ __forceinline__ int32_t row_min(const int32_t (&raw)[N]) {
    int32_t lo = raw[0];
#pragma unroll
    for (int i = 1; i < N; ++i) lo = min(lo, raw[i]);
    return lo;
}

// `lo` = row_min(raw): smaller than KC_CODE_NONE iff the group has absent cells.
template <int N, bool HAS_NC>
__device__ __forceinline__ void vote_core(const int32_t (&raw)[N], int32_t lo, int32_t none_code, int32_t &win_code,
                                          uint32_t &meta) {
    using M = typename MaskOf<N>::type;
    int32_t x[N];
    const uint32_t flip = (HAS_NC && none_code >= 0) ? ~(uint32_t)none_code : 0u;
    if (lo < KC_CODE_NONE) {  // rare: some candidate is not part of this node (nested payloads)
        int present = 0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const bool absent = raw[i] < KC_CODE_NONE;
            present += absent ? 0 : 1;
            const int32_t t = (int32_t)((uint32_t)raw[i] ^ ((uint32_t)(raw[i] >> 31) & flip));
            x[i] = absent ? KC_CODE_NONE : t;
        }
        meta = vote_scan<N, M>(x, present, win_code);
        return;
    }
    uint32_t non_voting = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if constexpr (HAS_NC)
            x[i] = (int32_t)((uint32_t)raw[i] ^ ((uint32_t)(raw[i] >> 31) & flip));  // -1 -> none_code when None votes
        else
            x[i] = raw[i];
        non_voting += (uint32_t)x[i] >> 31;
    }
    const int voters = N - (int)non_voting;
    const int32_t c = guess_mode<N>(x);
    if (c >= 0) {
        M eq = 0;
#pragma unroll
        for (int j = 0; j < N; ++j) eq |= (x[j] == c) ? (M(1) << j) : M(0);
        const int cnt = popc_m(eq);
        if (2 * cnt > voters) {
            win_code = c;
            meta = pack_meta(ffs_mask(eq) - 1, cnt, voters, N, KC_FLAG_HAS_VALUE);
            return;
        }
    }
    meta = vote_scan<N, M>(x, N, win_code);
}

// The field phase of a strided walk over groups: f is the field of the current group, and advance() moves it `step` groups
// on with one subtraction (f and step are both < n_fields).
struct FieldCursor {
    uint32_t f, step, n_fields;
    __device__ __forceinline__ void advance() {
        f += step;
        f = f >= n_fields ? f - n_fields : f;
    }
};

// field of group g without a 64-bit modulo: f = x - (x*magic >> 32)*F, exact for x < 2^16 (magic = 2^32/F + 1)
struct FieldMap {
    const int32_t *none_code;  // NULL => no field has voting Nones
    uint32_t n_fields;
    uint32_t magic;
    // x / n_fields and x % n_fields for x < n_fields + a few hundred (magic = 2^32 / n_fields + 1 does not fit for n_fields = 1)
    __device__ __forceinline__ uint32_t div_small(uint32_t x) const { return n_fields == 1u ? x : __umulhi(x, magic); }
    __device__ __forceinline__ uint32_t mod_small(uint32_t x) const { return x - div_small(x) * n_fields; }
    // a walk over units of UNIT consecutive groups that starts at unit `first` and advances `step` units at a time; these are
    // its only divisions
    template <int UNIT = 1, typename I>
    __device__ __forceinline__ FieldCursor cursor(I first, I step) const {
        return {(uint32_t)((first * UNIT) % n_fields), (uint32_t)((step * UNIT) % n_fields), n_fields};
    }
};

// ---------------------------------------------------------------- direct front-end

// Row g of n cells into registers; one overload per cell type.  NP = n rounded up to a power of two (compile-time register
// array); cells beyond n are padded absent.
template <int NP, bool VEC>
__device__ __forceinline__ void load_row(const int32_t *__restrict__ codes, int64_t g, int n, int32_t (&raw)[NP]) {
    if constexpr (VEC) {  // n == NP, rows are 16-byte aligned multiples of 16 bytes
        if constexpr (NP >= 4) {
            const int4 *p = reinterpret_cast<const int4 *>(codes + g * NP);
#pragma unroll
            for (int q = 0; q < NP / 4; ++q) {
                const int4 t = ldg_nc_v4(p + q);
                raw[4 * q + 0] = t.x;
                raw[4 * q + 1] = t.y;
                raw[4 * q + 2] = t.z;
                raw[4 * q + 3] = t.w;
            }
        } else if constexpr (NP == 2) {
            const int2 t = __ldg(reinterpret_cast<const int2 *>(codes + g * 2));
            raw[0] = t.x;
            raw[1] = t.y;
        } else {
            raw[0] = __ldg(codes + g);
        }
    } else {
        const int32_t *p = codes + g * n;
#pragma unroll
        for (int i = 0; i < NP; ++i) raw[i] = (i < n) ? __ldg(p + i) : KC_CODE_ABSENT;
    }
}

// Compact cells (int8).  Votes only need equality INSIDE a group, so a group can always be re-coded with local codes 0..n-1
// (< 64): one byte per cell (-1 None, -2 absent) is a lossless input format at a quarter of the bytes — what the end-to-end
// host path ships over PCIe.  A row of n = 16 cells is ONE 16-byte load per thread (a warp reads 512 contiguous bytes).
template <int NP, bool VEC>
__device__ __forceinline__ void load_row(const int8_t *__restrict__ codes, int64_t g, int n, int32_t (&raw)[NP]) {
    if constexpr (VEC && NP >= 4) {
        const uint32_t *p = reinterpret_cast<const uint32_t *>(codes + g * NP);
        uint32_t w[NP / 4];
        if constexpr (NP >= 16) {
#pragma unroll
            for (int q = 0; q < NP / 16; ++q) {
                const int4 t = ldg_nc_v4(reinterpret_cast<const int4 *>(p) + q);
                w[4 * q + 0] = (uint32_t)t.x;
                w[4 * q + 1] = (uint32_t)t.y;
                w[4 * q + 2] = (uint32_t)t.z;
                w[4 * q + 3] = (uint32_t)t.w;
            }
        } else if constexpr (NP == 8) {
            const uint2 t = __ldg(reinterpret_cast<const uint2 *>(p));
            w[0] = t.x;
            w[1] = t.y;
        } else {
            w[0] = __ldg(p);
        }
#pragma unroll
        for (int i = 0; i < NP; ++i) raw[i] = (int32_t)(int8_t)(w[i / 4] >> (8 * (i % 4)));
    } else {
        const int8_t *p = codes + g * n;
#pragma unroll
        for (int i = 0; i < NP; ++i) raw[i] = (i < n) ? (int32_t)__ldg(p + i) : KC_CODE_ABSENT;
    }
}

// Grid-stride, one group per thread per iteration, on Cell = int32_t or int8_t cells.  With PREFETCH the next iteration's
// row is requested before the current one is processed (twice the bytes in flight per thread, for ~NP more registers).
template <typename Cell, int NP, bool VEC, bool HAS_NC, bool PREFETCH>
__global__ void __launch_bounds__(256) vote_direct_kernel(const Cell *__restrict__ codes, int64_t n_groups, int n,
                                                          FieldMap fm, int32_t *__restrict__ win,
                                                          uint32_t *__restrict__ meta, const __grid_constant__ OutRoute mc) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    FieldCursor field = fm.cursor(g, stride);
    int32_t raw[NP];
    if (PREFETCH && g < n_groups) load_row<NP, VEC>(codes, g, n, raw);
    for (; g < n_groups; g += stride) {
        int32_t nxt[NP];
        if constexpr (PREFETCH) {
            if (g + stride < n_groups) load_row<NP, VEC>(codes, g + stride, n, nxt);
        } else {
            load_row<NP, VEC>(codes, g, n, raw);
        }
        int32_t nc = KC_CODE_NONE;
        if constexpr (HAS_NC) {
            nc = __ldg(fm.none_code + field.f);
            field.advance();
        }
        int32_t w;
        uint32_t m;
        vote_core<NP, HAS_NC>(raw, row_min<NP>(raw), nc, w, m);
        store_vote_result(win, meta, g, w, m, mc);
        if constexpr (PREFETCH) {
#pragma unroll
            for (int i = 0; i < NP; ++i) raw[i] = nxt[i];
        }
    }
}

// The same result as vote_core for very small groups, without guess / scan control flow: all pairwise equalities, the size
// of every cell's class, then the first-seen rule (a later class must be STRICTLY larger, cu:958,969) over the first cells of
// the classes.  Branch-free; N (N - 1) / 2 compares.  At n = 2 the HBM roofline leaves ~46 thread-instructions per group: the
// generic core's fixed cost (guess, equality pass, majority test, fall-through scan) is what bounded the small-n kernels.
template <int N, bool HAS_NC>
__device__ __forceinline__ void vote_core_small(const int32_t (&raw)[N], int32_t none_code, int32_t &win_code, uint32_t &meta) {
    const uint32_t flip = (HAS_NC && none_code >= 0) ? ~(uint32_t)none_code : 0u;
    int32_t x[N];
    uint32_t v[N], cnt[N], later[N];  // votes?  class size;  has an equal voting cell BEFORE it (not the class's first cell)
    uint32_t present = 0, voters = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const bool absent = raw[i] < KC_CODE_NONE;
        const int32_t t = HAS_NC ? (int32_t)((uint32_t)raw[i] ^ ((uint32_t)(raw[i] >> 31) & flip)) : raw[i];
        x[i] = absent ? KC_CODE_NONE : t;
        v[i] = x[i] >= 0 ? 1u : 0u;
        cnt[i] = v[i];
        later[i] = 0;
        present += absent ? 0u : 1u;
        voters += v[i];
    }
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
        for (int j = i + 1; j < N; ++j) {
            const uint32_t e = (x[i] == x[j]) ? (v[i] & v[j]) : 0u;
            cnt[i] += e;
            cnt[j] += e;
            later[j] |= e;
        }
    uint32_t best_cnt = 0, best_idx = 0, ties = 0;  // ties: classes (first cells) whose size equals the current best
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const uint32_t c = later[i] ? 0u : cnt[i];  // only the first cell of a class competes
        const bool gt = c > best_cnt;
        ties = gt ? 0u : ties + ((c == best_cnt && c != 0u) ? 1u : 0u);
        best_idx = gt ? (uint32_t)i : best_idx;
        best_cnt = gt ? c : best_cnt;
    }
    int32_t w = KC_CODE_NONE;
#pragma unroll
    for (int i = 0; i < N; ++i) w = (best_cnt != 0u && best_idx == (uint32_t)i) ? x[i] : w;
    win_code = w;
    meta = pack_meta(best_idx, best_cnt, voters, present, best_cnt ? (KC_FLAG_HAS_VALUE | (ties ? KC_FLAG_TIE : 0u)) : 0u);
}

// Small rows (n = 2, 4, 8): one group per thread leaves 8-32 bytes in flight per thread and a fixed cost per group that the
// few cells cannot amortise.  Here a thread owns GPT
// CONSECUTIVE groups = 64 bytes of cells (the access pattern of the n = 16 kernel: four 16-byte loads per thread, a warp
// covers 2 KB contiguous), the next 64 bytes are requested before these are processed, and the GPT results leave as 16-byte
// (GPT >= 4) or 8-byte vectors.  n_groups must be a multiple of GPT (the launcher sends the remainder to vote_direct_kernel).
template <int NP, int GPT, bool HAS_NC>
__global__ void __launch_bounds__(256) vote_multi_kernel(const int32_t *__restrict__ codes, int64_t n_units, FieldMap fm,
                                                         int32_t *__restrict__ win, uint32_t *__restrict__ meta) {
    static_assert(NP * GPT == 16, "a thread's unit is 64 bytes of cells");
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    FieldCursor field = fm.cursor<GPT>(u, stride);  // the field of the unit's first group
    int32_t raw[16];
    auto load = [&](int64_t unit, int32_t (&dst)[16]) {
        const int4 *p = reinterpret_cast<const int4 *>(codes) + unit * 4;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int4 t = ldg_nc_v4(p + q);
            dst[4 * q + 0] = t.x;
            dst[4 * q + 1] = t.y;
            dst[4 * q + 2] = t.z;
            dst[4 * q + 3] = t.w;
        }
    };
    if (u < n_units) load(u, raw);
    for (; u < n_units; u += stride) {
        int32_t nxt[16];
        if (u + stride < n_units) load(u + stride, nxt);
        int32_t w[GPT];
        uint32_t m[GPT];
#pragma unroll
        for (int j = 0; j < GPT; ++j) {
            int32_t x[NP];
#pragma unroll
            for (int i = 0; i < NP; ++i) x[i] = raw[j * NP + i];
            int32_t nc = KC_CODE_NONE;
            if constexpr (HAS_NC) {
                uint32_t fj = field.f + (uint32_t)j;  // consecutive groups are consecutive fields
                fj = fj >= fm.n_fields ? fm.mod_small(fj) : fj;
                nc = __ldg(fm.none_code + fj);
            }
            if constexpr (NP <= 4) vote_core_small<NP, HAS_NC>(x, nc, w[j], m[j]);
            else vote_core<NP, HAS_NC>(x, row_min<NP>(x), nc, w[j], m[j]);
        }
        if constexpr (HAS_NC) field.advance();
        if constexpr (GPT >= 4) {
#pragma unroll
            for (int q = 0; q < GPT / 4; ++q) {
                asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(win + u * GPT + 4 * q), "r"(w[4 * q]), "r"(w[4 * q + 1]),
                             "r"(w[4 * q + 2]), "r"(w[4 * q + 3])
                             : "memory");
                asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(meta + u * GPT + 4 * q), "r"(m[4 * q]), "r"(m[4 * q + 1]),
                             "r"(m[4 * q + 2]), "r"(m[4 * q + 3])
                             : "memory");
            }
        } else {
            asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(win + u * GPT), "r"(w[0]), "r"(w[1]) : "memory");
            asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(meta + u * GPT), "r"(m[0]), "r"(m[1]) : "memory");
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) raw[i] = nxt[i];
    }
}

// ---------------------------------------------------------------- TMA front-end

// Persistent kernel on WarpTiles (kc_common.cuh): lane l votes row l of the warp's current tile.
template <int N, int WARPS, int STAGES, bool HAS_NC>
__global__ void __launch_bounds__(WARPS * 32) vote_tma_kernel(const __grid_constant__ CUtensorMap tmap, uint32_t n_groups,
                                                              FieldMap fm, int32_t *__restrict__ win,
                                                              uint32_t *__restrict__ meta, const __grid_constant__ OutRoute mc) {
    WarpTiles<N * 4, WARPS, STAGES> tiles(&tmap, n_groups);
    tiles.start(L2Policy::evict_first);

    FieldCursor field = fm.cursor<32>((uint64_t)tiles.t, (uint64_t)tiles.step);  // the field of the tile's first group
    for (; tiles.t < tiles.n_tiles; tiles.next()) {
        const uint32_t tile = tiles.wait();
        int32_t raw[N];
        tiles.read_row(tile, raw);
        const int32_t lo = row_min<N>(raw);
        tiles.release((uint32_t)lo);
        const uint32_t g = tiles.t * 32 + tiles.lane;
        int32_t nc = KC_CODE_NONE;
        if constexpr (HAS_NC) {
            nc = __ldg(fm.none_code + fm.mod_small(field.f + tiles.lane));
            field.advance();
        }
        if (g < n_groups) {
            int32_t w;
            uint32_t m;
            vote_core<N, HAS_NC>(raw, lo, nc, w, m);
            store_vote_result(win, meta, g, w, m, mc);
        }
    }
}

}  // namespace kc
