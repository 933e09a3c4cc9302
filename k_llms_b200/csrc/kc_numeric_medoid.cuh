// kc_numeric_medoid.cuh — K5: similarity medoid of numeric groups, the primitive branch of the reference's ASYNC dispatcher
// (async_consensus_as_primitive, consensus_utils.py:1638-1688), which has no numeric clustering.
//
// Over the k non-None cells of a group: pairwise numerical_similarity (cu:827-841: math.isclose(rel_tol=0.01) -> 1.0, else the
// 1e-8 floor; for numbers this also covers generic_similarity's both-falsy rule and the == fallback), np.nanmean of every row
// of the k x k matrix (diagonal NaN), first argmax.  nanmean sums a copy with NaN -> 0, so the diagonal adds +0.0 in numpy's
// pairwise order (np_sum), then one IEEE division by k - 1.
//
// The row with the most close neighbours is NOT always the winner: rows with the same count differ in the last ulp depending
// on where the pairwise order meets the 1e-8 terms ([10, 10, 20, 20, 30] -> 20).  So every row sum is computed exactly and the
// means are compared as numpy compares them.
//
// Layout: a TEAM of lanes per group (team = n rounded up to a power of two, at most 32), 32 / team groups per warp.  The team
// compacts its group's non-None cells into shared memory (ballot + prefix count); lane i then sums rows i, i + team, ... and a
// shuffle reduction over the team picks the first maximum.  Every lane of a team reads the same cell at once (a broadcast).
#pragma once

#include "kc_internal.h"
#include "kc_numeric.cuh"  // np_sum, kNoneHi, kAbsentHi

namespace kc {

constexpr int kNumMedoidWarps = 4;

__global__ void __launch_bounds__(kNumMedoidWarps * 32) numeric_medoid_kernel(const double *__restrict__ cells, int64_t n_groups, int n,
                                                                              int team, int32_t *__restrict__ best,
                                                                              double *__restrict__ best_avg) {
    __shared__ double s_vals[kNumMedoidWarps][KC_MAX_CANDIDATES];
    const int lane_w = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tpw = 32 / team, lane = lane_w & (team - 1), t = lane_w / team;
    const uint32_t team_bits = team == 32 ? 0xFFFFFFFFu : ((1u << team) - 1u);
    const uint32_t below = (1u << lane) - 1u;  // the team's lanes before this one (team-local bit positions)
    double *vals = s_vals[warp] + t * team;    // a team of 32 owns all 64 slots; smaller teams hold n <= team cells
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t rounds = (n_groups + tpw - 1) / tpw;
    const double qnan = __longlong_as_double(0x7FF8000000000000LL);
    for (int64_t w = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); w < rounds; w += n_warps) {
        const int64_t g = w * tpw + t;
        const bool live = g < n_groups;
        // cells lane and lane + 32 (the second only for n > 32, where team = 32)
        double v0 = 0.0, v1 = 0.0;
        bool p0 = false, p1 = false;
        if (live && lane < n) {
            v0 = __ldg(cells + g * n + lane);
            const uint32_t h = (uint32_t)__double2hiint(v0);
            p0 = h != kNoneHi && h != kAbsentHi;
        }
        if (live && lane + 32 < n) {
            v1 = __ldg(cells + g * n + lane + 32);
            const uint32_t h = (uint32_t)__double2hiint(v1);
            p1 = h != kNoneHi && h != kAbsentHi;
        }
        const uint32_t b0 = (__ballot_sync(0xFFFFFFFFu, p0) >> (t * team)) & team_bits;
        const uint32_t b1 = (__ballot_sync(0xFFFFFFFFu, p1) >> (t * team)) & team_bits;
        const int k0 = __popc(b0), k = k0 + __popc(b1);
        __syncwarp();  // the previous round's readers are done with vals
        if (p0) vals[__popc(b0 & below)] = v0;
        if (p1) vals[k0 + __popc(b1 & below)] = v1;
        __syncwarp();
        double my_avg = -1.0;  // every mean is >= 1e-8
        int my_idx = 0x7FFFFFFF;
        if (k >= 2) {
            const double cnt = (double)(k - 1);  // the non-NaN entries of a row
            for (int i = lane; i < k; i += team) {
                const double xi = vals[i];
                const double tot = np_sum([&](int j) { return j == i ? 0.0 : (py_isclose(xi, vals[j]) ? 1.0 : kSimFloor); }, k);
                const double avg = __ddiv_rn(tot, cnt);
                if (avg > my_avg) {  // first maximum among this lane's rows (ascending i)
                    my_avg = avg;
                    my_idx = i;
                }
            }
        }
        for (int st = team >> 1; st >= 1; st >>= 1) {
            const double oa = __shfl_xor_sync(0xFFFFFFFFu, my_avg, st, team);
            const int oi = __shfl_xor_sync(0xFFFFFFFFu, my_idx, st, team);
            if (oa > my_avg || (oa == my_avg && oi < my_idx)) {
                my_avg = oa;
                my_idx = oi;
            }
        }
        if (live && lane == 0) {
            best[g] = k == 0 ? -1 : (k == 1 ? 0 : my_idx);
            best_avg[g] = k >= 2 ? my_avg : qnan;
        }
    }
}

}  // namespace kc
