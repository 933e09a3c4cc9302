// kc_extra.cuh — confidences (kc::confidence, kc_internal.h) and K3, the per-candidate logprob sum.
#pragma once

#include "kc_common.cuh"
#include "kc_internal.h"
#include "kc_vote.cuh"

namespace kc {

// One thread per group: the confidence the reference attaches to the group's consensus value.
__global__ void __launch_bounds__(256) confidence_kernel(const uint32_t *__restrict__ meta, int64_t n_groups, bool numeric,
                                                         const double *__restrict__ pvf_in, double *__restrict__ conf) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += stride) {
        const uint32_t m = __ldg(meta + g);
        const double pvf = pvf_in ? __ldg(pvf_in + g) : 1.0;
        conf[g] = confidence(m, numeric, pvf);
    }
}

// K3: one warp per sequence.  Lane l adds elements l, l+32, ... (coalesced 128-byte warp loads), then a
// xor butterfly 16,8,4,2,1 — the fixed order include/kllms_b200.h documents and oracle/consensus_oracle.c restates.
__global__ void __launch_bounds__(256) logprob_sum_kernel(const float *__restrict__ lp, const int64_t *__restrict__ offsets,
                                                          int64_t n_seq, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = warp; s < n_seq; s += n_warps) {
        const int64_t b = __ldg(offsets + s), e = __ldg(offsets + s + 1);
        float acc = 0.0f;
        for (int64_t i = b + lane; i < e; i += 32) acc = __fadd_rn(acc, __ldg(lp + i));
#pragma unroll
        for (int st = 16; st >= 1; st >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xFFFFFFFFu, acc, st));
        if (lane == 0) out[s] = acc;
    }
}

// K3, staged: sequences of a few dozen tokens leave a warp-per-sequence kernel with one or two elements per lane and
// ~25 instructions of bookkeeping per sequence.  Here a CTA copies the CONTIGUOUS
// token range of its T sequences into shared memory with 16-byte cp.async (coalesced, no register staging), then every
// thread sums ONE sequence in exactly the documented order: partial l = elements l, l+32, ... added left to right from
// +0.0f, then the tree the xor butterfly 16,8,4,2,1 forms (lane 0's view of it).  A tile whose tokens do not fit CAP
// floats (long sequences) falls back to the warp-per-sequence loop.
template <int T, int CAP>
__global__ void __launch_bounds__(T) logprob_sum_tile_kernel(const float *__restrict__ lp, const int64_t *__restrict__ offsets,
                                                             int64_t n_seq, float *__restrict__ out) {
    extern __shared__ __align__(16) float tok[];  // CAP + 4 floats
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t n_tiles = (n_seq + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t s0 = tile * T;
        const int cnt = (int)min((int64_t)T, n_seq - s0);
        // all four offset loads in flight together: the tile's range and this thread's sequence
        const int64_t t0 = __ldg(offsets + s0), t1 = __ldg(offsets + s0 + cnt);
        const int64_t my_b = __ldg(offsets + s0 + (tid < cnt ? tid : 0)), my_e = __ldg(offsets + s0 + (tid < cnt ? tid + 1 : 0));
        const int64_t t0a = t0 & ~int64_t(3);  // the copy starts at the 16-byte boundary at or below t0
        const int64_t span = t1 - t0a;
        if (span <= CAP) {
            const int n_vec = (int)(span >> 2);  // whole 16-byte pieces inside [t0a, t1)
            const uint32_t dst = smem_u32(tok);
            for (int v = tid; v < n_vec; v += T)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)v * 16u), "l"(lp + t0a + (int64_t)v * 4) : "memory");
            for (int i = (n_vec << 2) + tid; i < (int)span; i += T) tok[i] = __ldg(lp + t0a + i);  // < 4 stragglers
            asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
            __syncthreads();
            if (tid < cnt) {
                const int64_t b = my_b, e = my_e;
                const float *x = tok + (b - t0a);
                const int len = (int)(e - b);
                float p[32];
#pragma unroll
                for (int l = 0; l < 32; ++l) p[l] = 0.0f;
                for (int k = 0; k < len; k += 32) {
#pragma unroll
                    for (int l = 0; l < 32; ++l)
                        if (k + l < len) p[l] = __fadd_rn(p[l], x[k + l]);
                }
#pragma unroll
                for (int st = 16; st >= 1; st >>= 1) {
#pragma unroll
                    for (int l = 0; l < st; ++l) p[l] = __fadd_rn(p[l], p[l + st]);
                }
                out[s0 + tid] = p[0];
            }
            __syncthreads();  // the tile buffer is reused
        } else {
            for (int q = warp; q < cnt; q += T / 32) {
                const int64_t b = __ldg(offsets + s0 + q), e = __ldg(offsets + s0 + q + 1);
                float acc = 0.0f;
                for (int64_t i = b + lane; i < e; i += 32) acc = __fadd_rn(acc, __ldg(lp + i));
#pragma unroll
                for (int st = 16; st >= 1; st >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xFFFFFFFFu, acc, st));
                if (lane == 0) out[s0 + q] = acc;
            }
        }
    }
}

// ---------------------------------------------------------------- K3b: likelihood-weighted vote (self-defined spec)

// exp(x) for x <= 0, built only from single IEEE fp32 operations in a fixed order so that the C oracle
// (oracle/consensus_oracle.c: ko_exp_f32) reproduces it bit for bit: t = x*log2(e); k = floor(t + 0.5); f = t - k;
// 2^f by a degree-5 polynomial (Horner, separate multiply and add); scale by 2^k through the exponent field.
__device__ __forceinline__ float kexp(float x) {
    x = x < -87.0f ? -87.0f : x;
    const float t = __fmul_rn(x, 1.44269504f);
    const float k = floorf(__fadd_rn(t, 0.5f));
    const float f = __fadd_rn(t, -k);
    float p = 0.00133336f;
    p = __fadd_rn(__fmul_rn(p, f), 0.00961813f);
    p = __fadd_rn(__fmul_rn(p, f), 0.05550411f);
    p = __fadd_rn(__fmul_rn(p, f), 0.24022651f);
    p = __fadd_rn(__fmul_rn(p, f), 0.69314718f);
    p = __fadd_rn(__fmul_rn(p, f), 1.0f);
    return __fmul_rn(p, __int_as_float(((int)k + 127) << 23));
}

// One thread per group.  Candidate weight w_c = kexp(s_c - max_k s_k) with s = seq_logprob[record]; class weight =
// sum of its cells' weights in ascending candidate order (fp32); the heaviest class wins, ties -> first seen.
template <int NP>
__global__ void __launch_bounds__(128) weighted_vote_kernel(const int32_t *__restrict__ codes, const float *__restrict__ seq_lp,
                                                            int64_t n_groups, int n, FieldMap fm, bool has_nc,
                                                            int32_t *__restrict__ win, uint32_t *__restrict__ meta,
                                                            float *__restrict__ weight) {
    using M = typename MaskOf<NP>::type;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += stride) {
        const int64_t rec = g / fm.n_fields;
        const uint32_t field = (uint32_t)(g - rec * fm.n_fields);
        const int32_t nc = has_nc ? __ldg(fm.none_code + field) : KC_CODE_NONE;
        int32_t x[NP];
        float w[NP];
        float smax = -3.0e38f;
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            int32_t c = (i < n) ? __ldg(codes + g * n + i) : KC_CODE_ABSENT;
            const float s = (i < n) ? __ldg(seq_lp + rec * n + i) : -3.0e38f;
            w[i] = s;
            smax = (i < n && s > smax) ? s : smax;
            c = (c == KC_CODE_NONE) ? nc : c;           // None votes as none_code where it is >= 0
            x[i] = c < KC_CODE_NONE ? KC_CODE_NONE : c;  // absent cells never vote
        }
        M live = 0;
        int present = 0;
        float total = 0.0f;
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            w[i] = kexp(__fadd_rn(w[i], -smax));
            const bool absent = (i >= n) || __ldg(codes + g * n + (i < n ? i : 0)) < KC_CODE_NONE;
            present += absent ? 0 : 1;
            if (x[i] >= 0) {
                live |= M(1) << i;
                total = __fadd_rn(total, w[i]);
            }
        }
        const int voters = popc_m(live);
        float best_w = -1.0f;
        int best_idx = 0, best_cnt = 0;
        int32_t best_code = KC_CODE_NONE;
        bool tie = false;
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            if ((live >> i) & 1) {
                const int32_t c = x[i];
                M eq = 0;
                float cw = 0.0f;
#pragma unroll
                for (int j = i; j < NP; ++j) {
                    const bool e = x[j] == c;
                    eq |= e ? (M(1) << j) : M(0);
                    cw = e ? __fadd_rn(cw, w[j]) : cw;
                }
                if (cw > best_w) {
                    best_w = cw;
                    best_idx = i;
                    best_cnt = popc_m(eq);
                    best_code = c;
                    tie = false;
                } else if (cw == best_w) {
                    tie = true;
                }
                live &= ~eq;
            }
        }
        win[g] = best_code;
        meta[g] = pack_meta(best_idx, best_cnt, voters, present,
                            voters > 0 ? (KC_FLAG_HAS_VALUE | (tie ? KC_FLAG_TIE : 0u)) : 0u);
        weight[g] = voters > 0 ? __fdiv_rn(best_w, total) : 0.0f;
    }
}

// Candidate weights w_c = kexp(s_c - max_k s_k) of ONE record by a warp, lane = candidate: s_lo, s_hi = the sequence logprobs of
// candidates lane and lane + 32 (-3.0e38f where there is none).  Writes w[lane] (and w[lane + 32] for N > 32); returns the
// record's heaviest candidate, the first of the largest sums (N if there is none, e.g. all NaN).  The max is the fmaxf butterfly
// 16..1, so every lane holds the same one.
template <int N>
__device__ __forceinline__ int record_weights(float s_lo, float s_hi, float *w, uint32_t lane) {
    float smax = fmaxf(s_lo, s_hi);
#pragma unroll
    for (int st = 16; st >= 1; st >>= 1) smax = fmaxf(smax, __shfl_xor_sync(0xFFFFFFFFu, smax, st));
    if (N >= 32 || lane < N) w[lane] = kexp(__fadd_rn(s_lo, -smax));
    if (N > 32) w[lane + 32] = kexp(__fadd_rn(s_hi, -smax));
    const uint32_t b_lo = __ballot_sync(0xFFFFFFFFu, s_lo == smax), b_hi = __ballot_sync(0xFFFFFFFFu, N > 32 && s_hi == smax);
    return b_lo ? __ffs((int)b_lo) - 1 : (b_hi ? 31 + __ffs((int)b_hi) : N);
}

// Where every walk below stops.  Each class not summed yet sums a subset of the weights not consumed yet, so its fp32 sum is at
// most (total - consumed) up to rounding (< 64 * 2^-23 relative on each side); kWvSlack * total covers that.  A class below
// this bound can neither win nor tie.
constexpr float kWvSlack = 5e-5f;
__device__ __forceinline__ float wv_rest_bound(float total, float consumed) {
    return __fadd_rn(__fadd_rn(total, -consumed), __fmul_rn(total, kWvSlack));
}

// The weighted vote of ONE group by one thread: rawrow = the group's cells (code >= 0, KC_CODE_NONE, absent < KC_CODE_NONE), nc = the
// code None votes as (KC_CODE_NONE: it does not), w = the candidate weights of the group's record.  The outcome: the heaviest
// class (its cells' weights summed in ascending candidate order, fp32) wins, equal weights go to the class seen first (the
// smaller first index), `tie` says whether another class equals the winner.
template <int NP>
__device__ __forceinline__ void weighted_core(const int32_t (&rawrow)[NP], int32_t nc, const float *w, int32_t &out_code,
                                              uint32_t &out_meta, float &out_weight) {
    using M = typename MaskOf<NP>::type;
    int32_t x[NP];
    M live = 0;
    int present = 0;
    float total = 0.0f, wmax = -1.0f;
    int32_t cmax = KC_CODE_NONE;  // the code of this group's heaviest VOTING cell (first of equals)
#pragma unroll
    for (int i = 0; i < NP; ++i) {
        const int32_t raw = rawrow[i];
        int32_t c = (raw == KC_CODE_NONE) ? nc : raw;  // None votes as none_code where it is >= 0
        c = c < KC_CODE_NONE ? KC_CODE_NONE : c;        // absent cells never vote
        x[i] = c;
        present += raw < KC_CODE_NONE ? 0 : 1;
        if (c >= 0) {
            live |= M(1) << i;
            const float wi = w[i];
            total = __fadd_rn(total, wi);
            if (wi > wmax) {
                wmax = wi;
                cmax = c;
            }
        }
    }
    const int voters = popc_m(live);
    float best_w = -1.0f;
    int best_idx = 0, best_cnt = 0;
    int32_t best_code = KC_CODE_NONE;
    bool tie = false;
    float consumed = 0.0f;
    // Order of the walk: always the class of the heaviest cell still waiting (the first one: this group's heaviest
    // voting cell).  The outcome does not depend on the order (the heaviest class wins, equal weights go to the class
    // seen first = smaller first index, `tie` says whether another class equals the winner), but the COST does: a warp
    // loops until its slowest lane is done.  The heaviest voter's class usually holds more than half of the weight and
    // ends the walk at once; where it does not, going by weight makes the remainder shrink fastest.  (Round 1 walked
    // in first-seen order after the record's heaviest candidate: 4.3 class passes per warp, and it parked every
    // group's codes in a shared-memory plane to fetch the next class's code by a data-dependent index; here the pass
    // over the cells finds the next class itself — no shared memory for the codes at all.)
    int32_t c = cmax;
    while (live) {
        if (wv_rest_bound(total, consumed) < best_w) break;
        M eq = 0;
        float cw = 0.0f, nw = -1.0f;
        int32_t nc2 = KC_CODE_NONE;
#pragma unroll
        for (int j = 0; j < NP; ++j) {
            const bool e = x[j] == c;  // cells with this code that came earlier were consumed with their class
            const float wj = w[j];
            eq |= e ? (M(1) << j) : M(0);
            cw = e ? __fadd_rn(cw, wj) : cw;
            const bool waiting = !e && ((live >> j) & 1);
            if (waiting && wj > nw) {  // heaviest cell of the classes still waiting (first of equals)
                nw = wj;
                nc2 = x[j];
            }
        }
        const int i = ffs_mask(eq) - 1;  // the class's first cell
        if (cw > best_w) {
            best_w = cw;
            best_idx = i;
            best_cnt = popc_m(eq);
            best_code = c;
            tie = false;
        } else if (cw == best_w) {
            tie = true;
            if (i < best_idx) {  // an equally heavy class that was seen earlier
                best_idx = i;
                best_cnt = popc_m(eq);
                best_code = c;
            }
        }
        consumed = __fadd_rn(consumed, cw);
        live &= ~eq;
        c = nc2;
        if (c < 0) break;  // no waiting cell had a comparable weight (NaN logprobs: outside the spec); never spin
    }
    out_code = best_code;
    out_meta = pack_meta(best_idx, best_cnt, voters, present, voters > 0 ? (KC_FLAG_HAS_VALUE | (tie ? KC_FLAG_TIE : 0u)) : 0u);
    out_weight = voters > 0 ? __fdiv_rn(best_w, total) : 0.0f;
}

// K3b, weights once per record: the candidate weights depend on the record only, not on the field.  A CTA of T threads
// covers T consecutive groups (fields of a handful of records); its warps first compute the weights of those records into
// shared memory (record_weights), then every thread votes its group with the weights read from there.
template <int NP, int T>
__global__ void __launch_bounds__(T) weighted_vote_rec_kernel(const int32_t *__restrict__ codes, const float *__restrict__ seq_lp,
                                                              int64_t n_groups, int n, FieldMap fm, bool has_nc,
                                                              int32_t *__restrict__ win, uint32_t *__restrict__ meta,
                                                              float *__restrict__ weight) {
    extern __shared__ float wts[];  // [records of the tile][NP]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t n_tiles = (n_groups + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t g0 = tile * T, g1 = min(g0 + T, n_groups);
        const int64_t r0 = g0 / fm.n_fields, r1 = (g1 - 1) / fm.n_fields;
        for (int64_t r = r0 + warp; r <= r1; r += T / 32) {
            const float s_lo = (lane < n) ? __ldg(seq_lp + r * n + lane) : -3.0e38f;
            const float s_hi = (NP > 32 && lane + 32 < n) ? __ldg(seq_lp + r * n + lane + 32) : -3.0e38f;
            record_weights<NP>(s_lo, s_hi, wts + (r - r0) * NP, (uint32_t)lane);
        }
        __syncthreads();
        const int64_t g = g0 + tid;
        if (g < g1) {
            // record and field of this thread without a 64-bit division: offset inside the tile's first record
            const uint32_t fpos = (uint32_t)(g0 - r0 * fm.n_fields) + (uint32_t)tid;
            const uint32_t rec_local = fm.div_small(fpos);
            const uint32_t field = fpos - rec_local * fm.n_fields;
            const int32_t nc = has_nc ? __ldg(fm.none_code + field) : KC_CODE_NONE;
            const float *w = wts + rec_local * NP;
            // (requesting the row BEFORE the weights phase was tried: it keeps 32 more registers live across the barrier,
            // 67 -> 94, and the lost occupancy cost more than the overlap gained)
            int32_t rawrow[NP];
            if (n == NP) load_row<NP, true>(codes, g, n, rawrow);
            else load_row<NP, false>(codes, g, n, rawrow);
            weighted_core<NP>(rawrow, nc, w, win[g], meta[g], weight[g]);
        }
        __syncthreads();
    }
}

// ---- K3b, TMA front-end: first pass per lane, undecided groups by the whole warp

// What a lane knows about its group after ONE pass over the cells: the mapped codes, the total weight of the voting cells and the
// class of the record's heaviest candidate (the guess), summed in index order exactly as a walk pass would.
template <int N>
struct WvFirst {
    using M = typename MaskOf<N>::type;
    int32_t x[N];
    M eq_g;
    float total, cw_g;
    int32_t guess;
    int voters, present;
    bool decided;  // the guess's class holds a strict majority of the weight: it is the unique winner
};

template <int N>
__device__ __forceinline__ void wv_first_pass(const int32_t (&raw)[N], int32_t lo, int32_t nc, const float *w, int32_t graw, WvFirst<N> &f) {
    using M = typename MaskOf<N>::type;
    f.eq_g = 0;
    f.total = 0.0f;
    f.cw_g = 0.0f;
    if (lo >= 0) {
        // every cell votes with its own code (no None, no absent cell — the common row): 2-3 ALU instructions per cell
        f.guess = graw < 0 ? KC_CODE_NONE : graw;
        f.voters = f.present = N;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const float wi = w[i];
            const bool e = raw[i] == f.guess;
            f.x[i] = raw[i];
            f.total = __fadd_rn(f.total, wi);
            if (e) {
                f.eq_g |= M(1) << i;
                f.cw_g = __fadd_rn(f.cw_g, wi);
            }
        }
    } else {
        int32_t guess = (graw == KC_CODE_NONE) ? nc : graw;
        f.guess = guess < KC_CODE_NONE ? KC_CODE_NONE : guess;  // the heaviest candidate does not vote here: no guess
        M live = 0;
        int present = 0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int32_t r = raw[i];
            int32_t c = (r == KC_CODE_NONE) ? nc : r;  // None votes as none_code where it is >= 0
            c = c < KC_CODE_NONE ? KC_CODE_NONE : c;    // absent cells never vote
            f.x[i] = c;
            present += r < KC_CODE_NONE ? 0 : 1;
            if (c >= 0) {
                live |= M(1) << i;
                const float wi = w[i];
                f.total = __fadd_rn(f.total, wi);
                if (c == f.guess) {
                    f.eq_g |= M(1) << i;
                    f.cw_g = __fadd_rn(f.cw_g, wi);
                }
            }
        }
        f.voters = popc_m(live);
        f.present = present;
    }
    f.decided = f.guess >= 0 && f.cw_g > wv_rest_bound(f.total, f.cw_g);
}

// The general walk (see weighted_core) for ONE group by the WHOLE warp: lane j holds cells j and j + 32 of the owner's group.  A
// thread-per-group walk makes the warp wait for its slowest lane — a few percent of the groups are undecided after the first
// pass, but most warps hold one — and spends 32 lanes on one lane's work; here an undecided group costs ~150 warp instructions.
// Same visiting order (the class of the heaviest cell still waiting, first of equals), same class sums (index order, one
// rounding per addition), same tie rules: the result is bit-identical.  All arguments except `owner` are the OWNER's values.
template <int N>
__device__ __forceinline__ void wv_warp_walk(uint32_t lane, uint32_t owner, const WvFirst<N> &f, const float *wts, uint32_t rec_local, int WROW,
                                             int32_t &out_code, uint32_t &out_meta, float &out_weight) {
    constexpr uint32_t FULL = 0xFFFFFFFFu;
    // the owner's cells, one (two) per lane
    int32_t c_lo = KC_CODE_NONE, c_hi = KC_CODE_NONE;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const int32_t v = __shfl_sync(FULL, f.x[j], owner);
        if (lane == (uint32_t)(j & 31)) {
            if (j < 32) c_lo = v;
            else c_hi = v;
        }
    }
    const float *w = wts + __shfl_sync(FULL, rec_local, owner) * WROW;
    const float w_lo = w[lane], w_hi = N > 32 ? w[lane + 32] : 0.0f;
    const float total = __shfl_sync(FULL, f.total, owner);
    const int32_t guess = __shfl_sync(FULL, f.guess, owner);
    const float cw_g = __shfl_sync(FULL, f.cw_g, owner);
    uint32_t live_lo = __ballot_sync(FULL, c_lo >= 0), live_hi = N > 32 ? __ballot_sync(FULL, c_hi >= 0) : 0u;
    float best_w = -1.0f, consumed = 0.0f;
    int best_idx = 0, best_cnt = 0;
    int32_t best_code = KC_CODE_NONE;
    bool tie = false;
    if (guess >= 0) {  // the first pass summed the guess's class: it is the best so far
        const uint32_t g_lo = __ballot_sync(FULL, c_lo == guess), g_hi = N > 32 ? __ballot_sync(FULL, c_hi == guess) : 0u;
        best_w = cw_g;
        best_idx = g_lo ? __ffs((int)g_lo) - 1 : 31 + __ffs((int)g_hi);
        best_cnt = __popc(g_lo) + __popc(g_hi);
        best_code = guess;
        consumed = cw_g;
        live_lo &= ~g_lo;
        live_hi &= ~g_hi;
    }
    while (live_lo | live_hi) {
        if (wv_rest_bound(total, consumed) < best_w) break;
        // the heaviest cell still waiting, first of equals
        float mx = fmaxf(((live_lo >> lane) & 1u) ? w_lo : -1.0f, (N > 32 && ((live_hi >> lane) & 1u)) ? w_hi : -1.0f);
#pragma unroll
        for (int st = 16; st >= 1; st >>= 1) mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, st));
        const uint32_t a_lo = __ballot_sync(FULL, ((live_lo >> lane) & 1u) && w_lo == mx);
        const uint32_t a_hi = N > 32 ? __ballot_sync(FULL, ((live_hi >> lane) & 1u) && w_hi == mx) : 0u;
        if (!(a_lo | a_hi)) break;  // only NaN weights are left (NaN logprobs: outside the spec); never spin
        const int32_t c = a_lo ? __shfl_sync(FULL, c_lo, __ffs((int)a_lo) - 1) : __shfl_sync(FULL, c_hi, __ffs((int)a_hi) - 1);
        const uint32_t e_lo = __ballot_sync(FULL, c_lo == c), e_hi = N > 32 ? __ballot_sync(FULL, c_hi == c) : 0u;
        float cw = 0.0f;  // the class's weights in index order
        for (uint32_t m = e_lo; m; m &= m - 1) cw = __fadd_rn(cw, __shfl_sync(FULL, w_lo, __ffs((int)m) - 1));
        if (N > 32)
            for (uint32_t m = e_hi; m; m &= m - 1) cw = __fadd_rn(cw, __shfl_sync(FULL, w_hi, __ffs((int)m) - 1));
        const int i = e_lo ? __ffs((int)e_lo) - 1 : 31 + __ffs((int)e_hi);
        const int cnt = __popc(e_lo) + __popc(e_hi);
        if (cw > best_w) {
            best_w = cw;
            best_idx = i;
            best_cnt = cnt;
            best_code = c;
            tie = false;
        } else if (cw == best_w) {
            tie = true;
            if (i < best_idx) {  // an equally heavy class that was seen earlier
                best_idx = i;
                best_cnt = cnt;
                best_code = c;
            }
        }
        consumed = __fadd_rn(consumed, cw);
        live_lo &= ~e_lo;
        live_hi &= ~e_hi;
    }
    if (lane == owner) {
        out_code = best_code;
        out_meta = pack_meta(best_idx, best_cnt, f.voters, f.present, f.voters > 0 ? (KC_FLAG_HAS_VALUE | (tie ? KC_FLAG_TIE : 0u)) : 0u);
        out_weight = f.voters > 0 ? __fdiv_rn(best_w, total) : 0.0f;
    }
}

// x / n_fields for any 32-bit x without a division: the multiply-high by inv_fields = wv_inv_fields(n_fields) =
// floor(2^64 / n_fields) + 1, exact for n_fields >= 2 (n_fields = 1 takes x itself).
KC_HD inline uint64_t wv_inv_fields(uint32_t n_fields) { return n_fields > 1u ? ~uint64_t(0) / n_fields + 1u : 0u; }
__device__ __forceinline__ uint32_t wv_record_of(uint32_t x, const FieldMap &fm, uint64_t inv_fields) {
    return fm.n_fields == 1u ? x : (uint32_t)__umul64hi((uint64_t)x, inv_fields);
}

// One tile of the K3b TMA kernels, from the wait for the tile to the stores: wts = the warp's weight rows for this tile (row
// pitch WROW, the index of the record's heaviest candidate at w[N]), g0 = the tile's first group, r0 = its record.  `extra`
// goes to release(): what the re-arm copies next to the tile it requests.  `f` is the lane's first-pass state, declared by
// the kernel: declared here, nvvm promotes it to registers while it optimises this function on its own, before inlining, and
// both kernels compile to other SASS with more stack (ptxas -v: weighted_vote_rows_kernel 24/24 -> 36/36 bytes of spills,
// weighted_vote_tma_kernel<32,...> 64 -> 72 bytes of stack).
template <int N, int WROW, int WARPS, int STAGES, class Extra>
__device__ __forceinline__ void wv_tma_tile(const WarpTiles<N * 4, WARPS, STAGES> &tiles, const float *wts, uint32_t g0, uint32_t r0,
                                            uint32_t n_groups, const FieldMap &fm, bool has_nc, int32_t *win, uint32_t *meta,
                                            float *weight, const Extra &extra, WvFirst<N> &f) {
    const uint32_t lane = tiles.lane;
    const uint32_t tile = tiles.wait();
    int32_t raw[N];
    tiles.read_row(tile, raw);
    const uint32_t g = g0 + lane;
    const uint32_t fpos = (g0 - r0 * fm.n_fields) + lane;  // offset inside the tile's first record: < n_fields + 32
    const uint32_t rec_local = g < n_groups ? fm.div_small(fpos) : 0u;
    const float *wrow = wts + rec_local * WROW;
    // this group's cell of its record's heaviest candidate: read from the tile while the stage is still ours
    const int imax = __float_as_int(wrow[N]);
    int32_t graw = KC_CODE_NONE - 1;
    if (imax < N) {
        asm volatile("ld.shared.s32 %0, [%1];" : "=r"(graw) : "r"(tile + tiles.at((uint32_t)imax * 4u)));
    }
    // the release's shuffle also means that every lane has left the previous tile, whose weight slot `extra` may refill
    const int32_t lo = min(row_min<N>(raw), graw);
    tiles.release((uint32_t)lo, extra);
    bool undecided = false;
    int32_t o_code = KC_CODE_NONE;
    uint32_t o_meta = 0;
    float o_weight = 0.0f;
    if (g < n_groups) {
        const uint32_t field = fpos - rec_local * fm.n_fields;
        const int32_t nc = has_nc ? __ldg(fm.none_code + field) : KC_CODE_NONE;
        wv_first_pass<N>(raw, lo, nc, wrow, graw, f);
        undecided = !f.decided;
        if (f.decided) {
            o_code = f.guess;
            o_meta = pack_meta(ffs_mask(f.eq_g) - 1, popc_m(f.eq_g), f.voters, f.present, KC_FLAG_HAS_VALUE);
            o_weight = __fdiv_rn(f.cw_g, f.total);
        }
    }
    for (uint32_t todo = __ballot_sync(0xFFFFFFFFu, undecided); todo; todo &= todo - 1)
        wv_warp_walk<N>(lane, (uint32_t)__ffs((int)todo) - 1u, f, wts, rec_local, WROW, o_code, o_meta, o_weight);
    if (g < n_groups) {
        win[g] = o_code;
        meta[g] = o_meta;
        weight[g] = o_weight;
    }
}

// K3b with K1's TMA front-end (n in {32, 64} cells per group = 128 / 256 byte rows; WarpTiles, kc_common.cuh) instead of one
// 128-byte row per thread straight from global memory (latency-bound at 0.39 of the HBM peak: a warp's 32 rows are 32 separate
// lines per load instruction).  The weights of the tile's records (32 groups span 31 / n_fields + 2 records at most) are computed
// by the warp itself (record_weights) into its own shared-memory rows of kWRowTile<N> = N + 1 floats: the odd pitch puts lanes of
// different records in different banks, and the pad slot carries the index of the record's heaviest candidate, whose class
// wv_first_pass sums in its one pass (which decides most groups).  No block-wide barrier.
template <int N>
constexpr int kWRowTile = N + 1;
template <int N, int WARPS, int STAGES>
constexpr size_t weighted_vote_tma_smem(int rec_cap) {
    return WarpTiles<N * 4, WARPS, STAGES>::RING_BYTES + (size_t)WARPS * rec_cap * kWRowTile<N> * 4;
}

template <int N, int WARPS, int STAGES, int MIN_CTAS, bool PREFETCH>
__global__ void __launch_bounds__(WARPS * 32, MIN_CTAS) weighted_vote_tma_kernel(const __grid_constant__ CUtensorMap tmap, const float *__restrict__ seq_lp,
                                                                       uint32_t n_groups, FieldMap fm, bool has_nc, int rec_cap, uint64_t inv_fields,
                                                                       int32_t *__restrict__ win, uint32_t *__restrict__ meta,
                                                                       float *__restrict__ weight) {
    constexpr int WROW = kWRowTile<N>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    WarpTiles<N * 4, WARPS, STAGES> tiles(&tmap, n_groups);
    const uint32_t lane = tiles.lane;
    // the weight rows live behind the tiles of all warps
    float *wts = reinterpret_cast<float *>(smem_raw + (tiles.end() - smem_u32(smem_raw))) + (size_t)tiles.warp * rec_cap * WROW;
    tiles.start(L2Policy::evict_first);

    // The sequence logprobs of a tile's records are requested one tile AHEAD (a warp works through its tiles one after the other:
    // a global-memory round trip per tile in front of the weights would be exposed every time).  Up to PF records per tile are
    // prefetched (32 groups span 31 / n_fields + 2 records); wider tiles load them on the spot.
    constexpr int PF = 4;
    const bool prefetch = PREFETCH && rec_cap <= PF;
    float cur_lo[PF], cur_hi[PF], nxt_lo[PF], nxt_hi[PF];
    auto fetch = [&](uint32_t tt, float (&lo)[PF], float (&hi)[PF]) {
        const uint32_t a = tt * 32, b = min(a + 31u, n_groups - 1u);
        const uint32_t ra = wv_record_of(a, fm, inv_fields), rb = wv_record_of(b, fm, inv_fields);
#pragma unroll
        for (int k = 0; k < PF; ++k) {
            lo[k] = hi[k] = -3.0e38f;
            if (ra + k <= rb) {
                const float *s = seq_lp + (size_t)(ra + k) * N;
                lo[k] = __ldg(s + lane);
                if (N > 32) hi[k] = __ldg(s + lane + 32);
            }
        }
    };
    if (prefetch && tiles.t < tiles.n_tiles) fetch(tiles.t, cur_lo, cur_hi);

    for (; tiles.t < tiles.n_tiles; tiles.next()) {
        const uint32_t t = tiles.t;
        if (prefetch && t + tiles.step < tiles.n_tiles) fetch(t + tiles.step, nxt_lo, nxt_hi);
        // the weights of this tile's records, while the tile is still on its way
        const uint32_t g0 = t * 32, g_last = min(g0 + 31u, n_groups - 1u);
        const uint32_t r0 = wv_record_of(g0, fm, inv_fields), r_last = wv_record_of(g_last, fm, inv_fields);
        for (uint32_t r = r0; r <= r_last; ++r) {
            const float *s = seq_lp + (size_t)r * N;
            float s_lo, s_hi = -3.0e38f;
            if (prefetch) {
                const uint32_t k = r - r0;  // < PF
                s_lo = k == 0 ? cur_lo[0] : k == 1 ? cur_lo[1] : k == 2 ? cur_lo[2] : cur_lo[3];
                if (N > 32) s_hi = k == 0 ? cur_hi[0] : k == 1 ? cur_hi[1] : k == 2 ? cur_hi[2] : cur_hi[3];
            } else {
                s_lo = __ldg(s + lane);
                if (N > 32) s_hi = __ldg(s + lane + 32);
            }
            float *w = wts + (r - r0) * WROW;
            const int imax = record_weights<N>(s_lo, s_hi, w, lane);
            if (lane == 0) w[N] = __int_as_float(imax);
        }
        __syncwarp();
        WvFirst<N> f;
        wv_tma_tile<N, WROW>(tiles, wts, g0, r0, n_groups, fm, has_nc, win, meta, weight, NoExtraCopy{}, f);
        __syncwarp();  // the next tile's weights overwrite these rows
        if (prefetch) {
#pragma unroll
            for (int k = 0; k < PF; ++k) {
                cur_lo[k] = nxt_lo[k];
                cur_hi[k] = nxt_hi[k];
            }
        }
    }
}

// ---- K3b with the weights OUT of the tile loop.  A pre-pass writes, once per record, the row [w_0 .. w_{N-1}, index of the heaviest
// candidate, 3 pad words] (kWRowBulk<N> = N + 4 floats: rows stay 16-byte multiples and consecutive rows start 4 banks apart); the
// vote kernel fetches the rows of a tile's records with ONE cp.async.bulk next to the tile's tensor copy, completing on the same
// mbarrier, into one of kWSlots<STAGES> = STAGES + 1 slots per warp: the slot of the tile being voted is not the one the re-arm refills.
template <int N>
constexpr int kWRowBulk = N + 4;
template <int STAGES>
constexpr int kWSlots = STAGES + 1;
template <int N, int WARPS, int STAGES>
constexpr size_t weighted_vote_rows_smem(int rec_cap) {
    return WarpTiles<N * 4, WARPS, STAGES>::RING_BYTES + (size_t)WARPS * kWSlots<STAGES> * rec_cap * kWRowBulk<N> * 4;
}

// The weight-row pre-pass, one warp per record.  FULL: n == N candidates per record (N >= 32).  Otherwise N is a bucket (a
// power of two >= n): records of n sums each, the lanes from n on weigh nothing (-3.0e38f, as for the missing candidates of
// record_weights).
template <int N, bool FULL>
__device__ __forceinline__ void weight_rows(const float *__restrict__ seq_lp, int64_t n_records, int n, float *__restrict__ rows) {
    constexpr int WROW = kWRowBulk<N>;
    const uint32_t lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n_records; r += n_warps) {
        const float *s = seq_lp + r * (FULL ? N : n);
        const float s_lo = (FULL || (int)lane < n) ? __ldg(s + lane) : -3.0e38f;
        const float s_hi = (N > 32 && (FULL || (int)lane + 32 < n)) ? __ldg(s + lane + 32) : -3.0e38f;
        float *w = rows + r * WROW;
        const int imax = record_weights<N>(s_lo, s_hi, w, lane);
        if (lane < 4) w[N + lane] = lane == 0 ? __int_as_float(imax) : 0.0f;
    }
}

template <int N>
__global__ void __launch_bounds__(256) weight_rows_kernel(const float *__restrict__ seq_lp, int64_t n_records, float *__restrict__ rows) {
    static_assert(N >= 32, "every lane holds a candidate");
    weight_rows<N, true>(seq_lp, n_records, N, rows);
}

// the rows of records of n <= NP candidates (kc_weighted_vote_groups_i8)
template <int NP>
__global__ void __launch_bounds__(256) weight_rows_n_kernel(const float *__restrict__ seq_lp, int64_t n_records, int n,
                                                            float *__restrict__ rows) {
    weight_rows<NP, false>(seq_lp, n_records, n, rows);
}

template <int N, int WARPS, int STAGES, int MIN_CTAS>
__global__ void __launch_bounds__(WARPS * 32, MIN_CTAS) weighted_vote_rows_kernel(const __grid_constant__ CUtensorMap tmap, const float *__restrict__ wrows,
                                                                        uint32_t n_groups, FieldMap fm, bool has_nc, int rec_cap, uint64_t inv_fields,
                                                                        int32_t *__restrict__ win, uint32_t *__restrict__ meta,
                                                                        float *__restrict__ weight) {
    constexpr int WROW = kWRowBulk<N>, WSLOTS = kWSlots<STAGES>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    WarpTiles<N * 4, WARPS, STAGES> tiles(&tmap, n_groups);
    const uint32_t slot_bytes = (uint32_t)rec_cap * WROW * 4;
    const uint32_t my_rows = tiles.end() + tiles.warp * (WSLOTS * slot_bytes);                           // shared-space address
    const float *my_rows_p = reinterpret_cast<const float *>(smem_raw + (my_rows - smem_u32(smem_raw)));  // the same, generic
    // the weight rows of the records tile tt belongs to, into the weight slot of the warp's tile number j
    auto weight_rows = [&](uint32_t tt, uint32_t j) -> ExtraCopy {
        const uint32_t a = tt * 32, b = min(a + 31u, n_groups - 1u);
        const uint32_t ra = wv_record_of(a, fm, inv_fields), rb = wv_record_of(b, fm, inv_fields);
        return {wrows + (size_t)ra * WROW, my_rows + (j % WSLOTS) * slot_bytes, (rb - ra + 1u) * WROW * 4};
    };
    tiles.start(L2Policy::evict_first, weight_rows);

    for (; tiles.t < tiles.n_tiles; tiles.next()) {
        const uint32_t g0 = tiles.t * 32;
        const float *wts = my_rows_p + (tiles.it % WSLOTS) * (slot_bytes / 4);
        WvFirst<N> f;
        wv_tma_tile<N, WROW>(tiles, wts, g0, wv_record_of(g0, fm, inv_fields), n_groups, fm, has_nc, win, meta, weight, weight_rows, f);
    }
}

// ---- K3b over ragged records (kc_weighted_vote_groups_i8): group g belongs to record group_record[g], in any order, and a
// record has any number of groups — the shape a planner produces when records differ in their vote fields.  Cells are K1's
// int8 cells (kc_vote_i8: -1 None, -2 absent, local codes >= 0, no none_code table).  The weight rows [R][kWRowBulk<NP>] come
// from weight_rows_kernel<NP, n == NP>; one thread votes one group with weighted_core, reading its record's row from global
// memory (rows of the same record are shared by its groups: L1 / L2 hits).  A group whose record index is outside
// [0, n_records) gets no value (meta 0, weight 0).
template <int NP, bool VEC>
__global__ void __launch_bounds__(128) weighted_vote_groups_kernel(const int8_t *__restrict__ codes, int64_t n_groups, int n,
                                                                   const int32_t *__restrict__ group_record, int64_t n_records,
                                                                   const float *__restrict__ wrows, int32_t *__restrict__ win,
                                                                   uint32_t *__restrict__ meta, float *__restrict__ weight) {
    constexpr int WROW = kWRowBulk<NP>;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += stride) {
        const int32_t rec = __ldg(group_record + g);
        int32_t raw[NP];
        load_row<NP, VEC>(codes, g, n, raw);
        if (rec < 0 || rec >= n_records) {
            win[g] = KC_CODE_NONE;
            meta[g] = 0u;
            weight[g] = 0.0f;
            continue;
        }
        weighted_core<NP>(raw, KC_CODE_NONE, wrows + (int64_t)rec * WROW, win[g], meta[g], weight[g]);
    }
}

}  // namespace kc
