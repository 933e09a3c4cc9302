// kc_medoid.cuh — K4: similarity medoid of multi-word strings (SURVEY.md §8f-2).
//
// Replaces, for groups of strings, the fallback of consensus_as_primitive (reference consensus_utils.py:1221-1237):
// pairwise levenshtein_similarity (cu:745-761: 1 - dist/max_len on normalize_string()ed text, floored at 1e-8),
// np.nanmean of every row of the k x k matrix (diagonal NaN), first argmax.  One WARP per group:
//   1. lanes hash their strings; every string finds the first identical one before it (its class representative) —
//      candidates of one LLM field mostly agree, and a distance is needed only between DISTINCT strings;
//   2. one lane per distinct string builds its Myers match table (36 x u64) in shared memory, once per group;
//   3. lanes split the u(u-1)/2 pairs of distinct strings; each distance is Myers' bit-parallel algorithm with the
//      SHORTER string as the pattern: 32-bit words when it has <= 32 characters, one 64-bit word otherwise.  The caller
//      guarantees min(len_i, len_j) <= 64 for every pair (always true under the reference's default method, which sends
//      pairs of two long strings to the embeddings service instead, cu:813); groups that violate it stay on the host;
//      the similarity (cu:758-761) is stored once per pair of classes;
//   4. lane i sums row i in numpy's pairwise order (diagonal contributes +0.0, as nanmean's NaN->0 copy does) and
//      divides by the k-1 valid entries; a shuffle reduction picks the first maximum.
// Strings arrive normalised (lower-case [a-z0-9]); the host does normalize_string() and the final round(pvf*avg, 5).
#pragma once

#include "kc_common.cuh"
#include "kc_numeric.cuh"  // np_sum

namespace kc {

constexpr int kMedoidMaxN = 64;        // strings per group
constexpr int kMedoidMaxPattern = 64;  // the shorter string of every pair must fit one 64-bit word
constexpr int kAlphabet = 36;
constexpr int kPeqStride = 37;  // u64 per table: odd, so that lanes building different tables spread over the banks

__host__ __device__ __forceinline__ int alnum_index(uint32_t c) { return (int)c - (c > 64u ? 'a' - 10 : '0'); }

// read-only byte load: through the non-coherent cache on the device, a plain load in the host instantiation
__host__ __device__ __forceinline__ uint8_t ld_ro(const uint8_t *p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

// Match table of a pattern of l <= 64 normalised characters: bit q of tab[c] is set where pattern[q] is symbol c.
__host__ __device__ __forceinline__ void myers_table(uint64_t *tab, const uint8_t *__restrict__ s, int l) {
#ifdef __CUDA_ARCH__
#pragma unroll 4
#endif
    for (int c = 0; c < kAlphabet; ++c) tab[c] = 0;
    for (int q = 0; q < l; ++q) tab[alnum_index(ld_ro(s + q))] |= 1ull << q;
}

// Edit distance of a pattern of m characters (match table peq) against text t.  Myers 1999 in Hyyro's formulation.
template <typename W>
__host__ __device__ __forceinline__ int myers(const uint64_t *peq, int m, const uint8_t *__restrict__ t, int tn) {
    W pv = ~W(0), mv = 0;
    int score = m;
    const int sh = m - 1;
    for (int k = 0; k < tn; ++k) {
        const W eq = (W)peq[alnum_index(ld_ro(t + k))];
        const W xv = eq | mv;
        const W xh = (((eq & pv) + pv) ^ pv) | eq;
        W ph = mv | ~(xh | pv);
        W mh = pv & xh;
        score += (int)((ph >> sh) & 1) - (int)((mh >> sh) & 1);
        ph = (ph << 1) | W(1);
        mh <<= 1;
        pv = mh | ~(xv | ph);
        mv = ph & xv;
    }
    return score;
}

// Per-warp shared memory for groups of at most `kmax` strings.
struct MedoidSmem {
    static __host__ __device__ size_t bytes(int kmax) {
        return (size_t)kmax * kPeqStride * 8 + (size_t)kmax * kmax * 8 + (size_t)kMedoidMaxN * (4 + 4 + 4 + 1 + 1 + 1) + 64;
    }
};

// chars: all strings back to back; str_off[s]..str_off[s+1] string s; grp_off[g]..grp_off[g+1] the strings of group g.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) medoid_kernel(const uint8_t *__restrict__ chars, const int32_t *__restrict__ str_off,
                                                            const int32_t *__restrict__ grp_off, int64_t n_groups, int kmax,
                                                            int32_t *__restrict__ best_idx, double *__restrict__ best_avg, int method) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t per_warp = (MedoidSmem::bytes(kmax) + 15) & ~size_t(15);
    uint8_t *wbase = smem_raw + (size_t)warp * per_warp;
    uint64_t *peq = reinterpret_cast<uint64_t *>(wbase);                 // [u][kPeqStride]
    double *sim = reinterpret_cast<double *>(peq + (size_t)kmax * kPeqStride);  // [u][kmax] similarity of two classes
    int32_t *s_off = reinterpret_cast<int32_t *>(sim + (size_t)kmax * kmax);  // [64] first character
    int32_t *s_len = s_off + kMedoidMaxN;                                 // [64]
    uint32_t *s_hash = reinterpret_cast<uint32_t *>(s_len + kMedoidMaxN);  // [64]
    uint8_t *s_cls = reinterpret_cast<uint8_t *>(s_hash + kMedoidMaxN);    // [64] string -> index of its class
    uint8_t *s_uniq = s_cls + kMedoidMaxN;                                     // [u] class -> first string of the class
    uint8_t *s_rep = s_uniq + kMedoidMaxN;                                     // [64] string -> first identical string

    const int64_t gw = (int64_t)blockIdx.x * WARPS + warp;
    const int64_t gstep = (int64_t)gridDim.x * WARPS;
    for (int64_t g = gw; g < n_groups; g += gstep) {
        const int s0 = __ldg(grp_off + g), k = __ldg(grp_off + g + 1) - s0;
        // 1. offsets, lengths, hashes (FNV-1a; only a filter: equality is confirmed character by character)
        for (int i = lane; i < k; i += 32) {
            const int o = __ldg(str_off + s0 + i), l = __ldg(str_off + s0 + i + 1) - o;
            uint32_t h = 2166136261u;
            for (int q = 0; q < l; ++q) h = (h ^ __ldg(chars + o + q)) * 16777619u;
            s_off[i] = o;
            s_len[i] = l;
            s_hash[i] = h;
        }
        __syncwarp();
        bool matched = false;  // every string found its representative through the hash match below
        if (k <= 32) {
            const bool live = lane < k;
            const uint32_t key = live ? (s_hash[lane] ^ ((uint32_t)s_len[lane] * 0x9E3779B1u)) : (0xFFFFFFFFu - lane);
            const int rep = __ffs(__match_any_sync(0xFFFFFFFFu, key)) - 1;  // lowest lane with the same (hash, length)
            bool same = true;
            if (live && rep != lane) {
                const int o = s_off[lane], orep = s_off[rep], l = s_len[lane];
                const uint8_t *pa = chars + o, *pb = chars + orep;
                uint32_t diff = s_len[rep] == l ? 0u : 1u;  // no early exit: equal hashes almost always mean equal strings
                int q = 0;
                if (diff == 0) {
                    for (; q + 4 <= l; q += 4)
                        diff |= (uint32_t)(__ldg(pa + q) ^ __ldg(pb + q)) | (uint32_t)(__ldg(pa + q + 1) ^ __ldg(pb + q + 1)) |
                                (uint32_t)(__ldg(pa + q + 2) ^ __ldg(pb + q + 2)) | (uint32_t)(__ldg(pa + q + 3) ^ __ldg(pb + q + 3));
                    for (; q < l; ++q) diff |= (uint32_t)(__ldg(pa + q) ^ __ldg(pb + q));
                }
                same = diff == 0;
            }
            matched = __all_sync(0xFFFFFFFFu, same);  // a hash collision sends the group to the exact scan
            if (matched && live) s_rep[lane] = (uint8_t)rep;
        }
        for (int i = lane; i < k && !matched; i += 32) {
            const int o = s_off[i], l = s_len[i];
            const uint32_t h = s_hash[i];
            int rep = i;
            for (int j = 0; j < i; ++j) {
                if (s_hash[j] == h && s_len[j] == l) {
                    const int oj = s_off[j];
                    int q = 0;
                    while (q < l && __ldg(chars + o + q) == __ldg(chars + oj + q)) ++q;
                    if (q == l) {
                        rep = j;
                        break;
                    }
                }
            }
            s_rep[i] = (uint8_t)rep;
        }
        __syncwarp();
        // class numbering in first-seen order
        int u = 0;
        for (int base = 0; base < k; base += 32) {
            const int i = base + lane;
            const bool first = i < k && s_rep[i] == i;
            const uint32_t mask = __ballot_sync(0xFFFFFFFFu, first);
            if (first) {
                const int c = u + __popc(mask & ((1u << lane) - 1u));
                s_uniq[c] = (uint8_t)i;
                s_cls[i] = (uint8_t)c;
            }
            u += __popc(mask);
        }
        __syncwarp();
        for (int i = lane; i < k; i += 32)
            if (s_rep[i] != i) s_cls[i] = s_cls[s_rep[i]];  // representatives already hold their own class (and only they are read)
        // 2. match tables of the distinct strings that can be a pattern
        for (int a = lane; a < u; a += 32) {
            const int i = s_uniq[a], o = s_off[i], l = s_len[i];
            uint64_t *tab = peq + (size_t)a * kPeqStride;
            if (method == 1) {  // jaccard_similarity (cu:720-742): the SET of characters, one bit per symbol of [a-z0-9]
                uint64_t set = 0;
                for (int q = 0; q < l; ++q) set |= 1ull << alnum_index(__ldg(chars + o + q));
                tab[0] = set;
            } else if (method == 0 && l <= kMedoidMaxPattern) {
                myers_table(tab, chars + o, l);
            }
            sim[a * kmax + a] = 1.0;  // identical strings: 1 - 0/max_len, or the empty-pair rule cu:756-757
        }
        __syncwarp();
        // 3. distances between distinct strings
        const int n_pairs = u * (u - 1) / 2;
        for (int p = lane; p < n_pairs; p += 32) {
            int a = 0, rem = p;  // (a, b), a < b, from the linear index over the upper triangle
            while (rem >= u - 1 - a) {
                rem -= u - 1 - a;
                ++a;
            }
            const int b = a + 1 + rem;
            int pa = a, ta = b;  // pattern = the shorter string
            if (s_len[s_uniq[a]] > s_len[s_uniq[b]]) {
                pa = b;
                ta = a;
            }
            const int m = s_len[s_uniq[pa]], to = s_off[s_uniq[ta]], tl = s_len[s_uniq[ta]];
            if (method == 1) {  // |A & B| / |A | B| on the character sets; distinct strings, so the union is not empty
                const uint64_t sa = peq[(size_t)a * kPeqStride], sb = peq[(size_t)b * kPeqStride];
                double sv = __ddiv_rn((double)__popcll(sa & sb), (double)__popcll(sa | sb));
                sv = sv > 1e-8 ? sv : 1e-8;
                sim[a * kmax + b] = sv;
                sim[b * kmax + a] = sv;
                continue;
            }
            int d;
            if (method == 2) {  // hamming_similarity (cu:676-717): position by position, the shorter string padded with ' '
                const int po = s_off[s_uniq[pa]];
                d = tl - m;  // a pad never equals an alphanumeric character
                for (int q = 0; q < m; ++q) d += __ldg(chars + po + q) != __ldg(chars + to + q) ? 1 : 0;
            } else if (m == 0)
                d = tl;
            else if (m <= 32)
                d = myers<uint32_t>(peq + (size_t)pa * kPeqStride, m, chars + to, tl);
            else  // m <= kMedoidMaxPattern by contract
                d = myers<uint64_t>(peq + (size_t)pa * kPeqStride, m, chars + to, tl);
            // cu:758-761; tl is the longer length (> 0, the strings differ)
            double sv = __dadd_rn(1.0, -__ddiv_rn((double)d, (double)tl));
            sv = sv > 1e-8 ? sv : 1e-8;
            sim[a * kmax + b] = sv;
            sim[b * kmax + a] = sv;
        }
        __syncwarp();
        // 4. row means and the first maximum
        double my_avg = -1.0;
        int my_idx = 0x7FFFFFFF;
        for (int i = lane; i < k; i += 32) {
            const double *srow = sim + (int)s_cls[i] * kmax;
            const double tot = np_sum([&](int j) { return j == i ? 0.0 : srow[s_cls[j]]; },  // nanmean: NaN -> 0 copy
                                      k);
            const double avg = __ddiv_rn(tot, (double)(k - 1));
            if (avg > my_avg) {  // first maximum within this lane's rows (ascending i)
                my_avg = avg;
                my_idx = i;
            }
        }
#pragma unroll
        for (int st = 16; st >= 1; st >>= 1) {
            const double oa = __shfl_xor_sync(0xFFFFFFFFu, my_avg, st);
            const int oi = __shfl_xor_sync(0xFFFFFFFFu, my_idx, st);
            if (oa > my_avg || (oa == my_avg && oi < my_idx)) {
                my_avg = oa;
                my_idx = oi;
            }
        }
        if (lane == 0) {
            best_idx[g] = my_idx;
            best_avg[g] = my_avg;
        }
        __syncwarp();
    }
}

}  // namespace kc
