// kc_common.cuh — sm_90a PTX helpers shared by the consensus kernels: mbarrier, TMA (cp.async.bulk.tensor) and the
// warp-private tile pipeline built on them, streaming stores, the packed result word.  No libraries; inline PTX only.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/kllms_b200.h"

namespace kc {

constexpr int kMaxN = KC_MAX_CANDIDATES;

__host__ __device__ __forceinline__ uint32_t pack_meta(uint32_t idx, uint32_t support, uint32_t nn, uint32_t present,
                                                       uint32_t flags) {
    return (idx & 0x3Fu) | ((support & 0x7Fu) << 6) | ((nn & 0x7Fu) << 13) | ((present & 0x7Fu) << 20) |
           ((flags & 0x1Fu) << 27);
}

// ---------------------------------------------------------------- shared-memory addresses, mbarrier (32-bit shared-space addresses)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}

// make mbarrier.init visible to the async (TMA) proxy
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "KC_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra KC_DONE_%=;\n\t"
        "bra KC_WAIT_%=;\n\t"
        "KC_DONE_%=:\n\t"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}

// ---------------------------------------------------------------- TMA: 2-D tiled tensor load, global -> swizzled smem

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// evict-first L2 policy for read-once streams
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

// Input tiles of a kernel that is NOT bandwidth-bound: normal priority, so that its result lines (also normal) are
// evicted — written back — while it runs.  With evict-first inputs the results outlive the kernel as up to an L2's worth
// of dirty lines and are written back under the next kernel's input stream.
__device__ __forceinline__ uint64_t policy_evict_normal() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap *map, int32_t c0, int32_t c1, uint32_t bar,
                                            uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], "
        "[%4], %5;" ::"r"(smem_dst),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar), "l"(policy)
        : "memory");
}

// contiguous bytes, global -> smem (16-byte aligned, a multiple of 16 bytes)
__device__ __forceinline__ void bulk_load_1d(uint32_t smem_dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
                 "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
                 : "memory");
}

// 16 bytes from a shared-space address
__device__ __forceinline__ int4 lds_v4(uint32_t addr) {
    int4 r;
    asm volatile("ld.shared.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}

// ---------------------------------------------------------------- the warp-private tile pipeline of the TMA front-ends

template <int ROW_BYTES>
struct Swizzle {  // TMA swizzle mode for a row of ROW_BYTES (rows wider than 128 B are split into 128 B box rows)
    static constexpr uint32_t kMask = ROW_BYTES >= 128 ? 7u : (ROW_BYTES == 64 ? 3u : 1u);
    __device__ static __forceinline__ uint32_t apply(uint32_t off) { return off ^ (((off >> 7) & kMask) << 4); }
};

// A further copy that lands on a tile's barrier next to the tile: `bytes` from `src` to the shared-space address `dst`;
// none if `src` is null.
struct ExtraCopy {
    const void *src;
    uint32_t dst, bytes;
};
struct NoExtraCopy {
    __device__ ExtraCopy operator()(uint32_t, uint32_t) const { return {nullptr, 0u, 0u}; }
};

enum class L2Policy { evict_first, evict_normal };

// Persistent kernels, warp-private pipelines.  Global warp w owns warp-tiles w, w + W, ... (W = warps in the grid); a
// warp-tile is 32 consecutive rows of ROW_BYTES (one group each) and lane l owns row l.  Each warp keeps STAGES tiles in
// flight in its own ring of swizzled shared-memory tiles: lane 0 arms the stage's mbarrier with the tile's byte count and
// issues one cp.async.bulk.tensor.2d; all lanes wait on the barrier and pull their row with swizzled (bank-conflict-free)
// LDS; release() hands the stage back for the tile STAGES ahead before the warp computes.  Out-of-range rows of the last
// tile are zero-filled by TMA and never stored.  There is no __syncthreads(): warps never wait for each other.  All indices
// are 32-bit: the launchers cut the input into slabs of < 2^28 groups.
//
//     WarpTiles<ROW_BYTES, WARPS, STAGES> tiles(&tmap, n_groups);
//     tiles.start(L2Policy::evict_first);
//     for (; tiles.t < tiles.n_tiles; tiles.next()) {
//         const uint32_t tile = tiles.wait();   // LDS at tile + tiles.at(byte of the row)
//         tiles.release(dep);                   // dep: computed from every load of the tile
//         ...                                   // group tiles.t * 32 + lane, from registers
//     }
//
// The dynamic shared memory holds the WARPS rings from its first 1024-byte boundary on; a kernel keeps its own data
// from end() on.
template <int ROW_BYTES, int WARPS, int STAGES>
struct WarpTiles {
    static constexpr uint32_t BOX_ROWS_PER_GROUP = ROW_BYTES > 128 ? ROW_BYTES / 128 : 1;
    static constexpr uint32_t TILE_BYTES = 32 * ROW_BYTES;
    // dynamic shared memory up to end(): the WARPS rings and the slack for aligning them to 1024 bytes
    static constexpr uint32_t RING_BYTES = 1024 + WARPS * STAGES * TILE_BYTES;
    static_assert(TILE_BYTES % 1024 == 0, "warp tile must keep the swizzle atom alignment");
    static_assert((STAGES & (STAGES - 1)) == 0, "STAGES must be a power of two");

    const CUtensorMap *map;
    uint32_t lane, warp;
    uint32_t base, ring, bar;  // shared-space addresses: all rings, this warp's ring, this warp's STAGES barriers
    uint32_t t, step, n_tiles;  // the current tile; the walk
    uint32_t it = 0;            // tiles done: stage it % STAGES, barrier phase (it / STAGES) & 1
    uint64_t policy = 0;        // lane 0's

    __device__ __forceinline__ WarpTiles(const CUtensorMap *tmap, uint32_t n_groups) : map(tmap) {
        extern __shared__ __align__(1024) uint8_t smem_raw[];
        __shared__ __align__(8) uint64_t full_bar[WARPS * STAGES];
        lane = threadIdx.x & 31;
        warp = __shfl_sync(0xFFFFFFFFu, threadIdx.x >> 5, 0);  // warp-uniform by construction
        base = (smem_u32(smem_raw) + 1023u) & ~1023u;
        ring = base + warp * (STAGES * TILE_BYTES);
        bar = smem_u32(full_bar) + warp * (STAGES * 8);
        n_tiles = (n_groups + 31u) >> 5;
        t = blockIdx.x * WARPS + warp;
        step = gridDim.x * WARPS;
    }

    // lane 0 sets up the barriers and requests the first STAGES tiles
    template <class Extra = NoExtraCopy>
    __device__ __forceinline__ void start(L2Policy l2, const Extra &extra = {}) {
        if (lane == 0) {
            tma_prefetch_desc(map);
#pragma unroll
            for (int s = 0; s < STAGES; ++s) mbar_init(bar + s * 8, 1);
            fence_barrier_init();
            policy = l2 == L2Policy::evict_first ? policy_evict_first() : policy_evict_normal();
#pragma unroll
            for (int s = 0; s < STAGES; ++s) {
                const uint32_t ts = t + (uint32_t)s * step;
                if (ts < n_tiles) arm(ts, (uint32_t)s, 0u, extra);
            }
        }
        __syncwarp();
    }

    // waits for the current tile; its shared-space address
    __device__ __forceinline__ uint32_t wait() const {
        const uint32_t s = it & (STAGES - 1), tile = ring + s * TILE_BYTES;  // before the wait: LDS can issue right after it
        mbar_wait(bar + s * 8, (it / STAGES) & 1);
        return tile;
    }

    // swizzled offset of byte `byte` of this lane's row inside a tile
    __device__ __forceinline__ uint32_t at(uint32_t byte) const { return Swizzle<ROW_BYTES>::apply(lane * ROW_BYTES + byte); }

    // this lane's row of 4-byte cells from the tile at `tile`, 16 bytes per load
    __device__ __forceinline__ void read_row(uint32_t tile, int32_t (&raw)[ROW_BYTES / 4]) const {
#pragma unroll
        for (int q = 0; q < ROW_BYTES / 16; ++q) {
            const int4 v4 = lds_v4(tile + at(q * 16));
            raw[4 * q + 0] = v4.x;
            raw[4 * q + 1] = v4.y;
            raw[4 * q + 2] = v4.z;
            raw[4 * q + 3] = v4.w;
        }
    }

    // Hands the current stage back: lane 0 requests the tile STAGES ahead into it.  Every row must be in registers first.
    // `dep` depends on every load the lane made from the tile, a warp instruction issues only when its operands are ready
    // in every lane, and the shuffle is one: `order` is 0 on lane 0 but only the hardware knows it (a shuffle result), so
    // folding it into the TMA coordinate gives the copy a true register dependency on the loaded data, which neither nvvm
    // nor ptxas can schedule away.
    template <class Extra = NoExtraCopy>
    __device__ __forceinline__ void release(uint32_t dep, const Extra &extra = {}) const {
        const uint32_t order = __shfl_sync(0xFFFFFFFFu, dep, 0) ^ dep;
        const uint32_t tn = t + STAGES * step;
        if (lane == 0 && tn < n_tiles) arm(tn, it + STAGES, order, extra);
    }

    __device__ __forceinline__ void next() {
        t += step;
        ++it;
    }

    // first shared-space address past the rings of all warps
    __device__ __forceinline__ uint32_t end() const { return base + WARPS * STAGES * TILE_BYTES; }

    // tile `tt`, the warp's tile number `j` (stage j % STAGES), plus what `extra(tt, j)` asks for, on the stage's barrier
    template <class Extra>
    __device__ __forceinline__ void arm(uint32_t tt, uint32_t j, uint32_t dep, const Extra &extra) const {
        const uint32_t s = j & (STAGES - 1), b = bar + s * 8;
        const ExtraCopy x = extra(tt, j);
        mbar_arrive_expect_tx(b, TILE_BYTES + x.bytes);
        tma_load_2d(ring + s * TILE_BYTES, map, 0, (int32_t)(tt * 32 * BOX_ROWS_PER_GROUP + dep), b, policy);
        if (x.src) bulk_load_1d(x.dst, x.src, x.bytes, b);
    }
};

// ---------------------------------------------------------------- global memory: streaming loads / stores

// read-only path, default L1 allocation: a thread's neighbouring 16-byte pieces share 32-byte sectors, so the
// second piece should hit L1 instead of going back to L2
__device__ __forceinline__ int4 ldg_nc_v4(const void *p) {
    int4 r;
    asm volatile("ld.global.nc.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// Result stores.  mc == true: `p` is an NVSwitch MULTICAST address (CUDA multicast object mapped on every GPU of
// the group); multimem.st makes the switch replicate the store into each GPU's copy of the buffer — the all-gather
// of the outputs happens inside the producing kernel, tile by tile, instead of in a separate collective.
// Where a kernel's results go.
//   LOCAL     plain stores (L1 no-allocate) to the given addresses;
//   MULTIMEM  the addresses are NVSwitch multicast addresses: multimem.st, the switch replicates every store into all
//             GPUs' copies — also back into the sender's own, so every GPU RECEIVES world x its share;
//   PEERS     the addresses are local and lie in a buffer that n_peers other GPUs map as well (symmetric memory): one
//             local store plus one store per peer at address + delta[k] (P2P over NVLink).  Each GPU receives only
//             (world - 1) shares and sends as many: less ingress than multicast, the better trade on full-duplex links.
//   PEERS_PACKED  (votes) the full result (winning code, result word) stays in LOCAL arrays — the owning rank's decoder
//             needs the first-seen index in it — and ONE packed word code:18 | support:7 | present:7, everything a remote
//             consumer needs for the value and its confidence, goes to `packed` (local + peers): 4 instead of 8 bytes per
//             vote field over NVLink.  A winning code >= 2^18 sets *overflow (the caller then falls back to PEERS).
struct OutRoute {
    uint32_t mode;       // KC_OUT_LOCAL / KC_OUT_MULTIMEM / KC_OUT_PEERS / 3 = PEERS_PACKED / 4 = WIRE (full result + local wire word, kc_push.cuh)
    int32_t n_peers;     // PEERS*, only
    long long delta[7];  // byte offsets local address -> the same address in peer k's mapping
    uint32_t *packed;    // PEERS_PACKED: local address (inside the shared buffer) of the packed vote words
    uint32_t *overflow;  // PEERS_PACKED / WIRE: device flag
    uint32_t wire_wide;  // WIRE (mode 4): 0 = u16 words code:6|support:5|present:5, 1 = u32 words code:18|support:7|present:7
    __host__ __device__ bool local() const { return mode == 0; }
};

// the P2P copies, out of line: the local path pays one uniform compare per store for them
__device__ __noinline__ void store_peers_u32(void *p, uint32_t v, const OutRoute &r) {
    for (int k = 0; k < r.n_peers; ++k)
        asm volatile("st.global.u32 [%0], %1;" ::"l"(reinterpret_cast<char *>(p) + r.delta[k]), "r"(v) : "memory");
}
__device__ __noinline__ void store_peers_f64(void *p, double v, const OutRoute &r) {
    for (int k = 0; k < r.n_peers; ++k)
        asm volatile("st.global.f64 [%0], %1;" ::"l"(reinterpret_cast<char *>(p) + r.delta[k]), "d"(v) : "memory");
}

__device__ __forceinline__ void store_local_u32(void *p, uint32_t v) {
    asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void store_local_f64(void *p, double v) {
    asm volatile("st.global.L1::no_allocate.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

__device__ __forceinline__ void store_out_u32(void *p, uint32_t v, const OutRoute &r) {
    if (r.mode == 1u) {
        asm volatile("multimem.st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
    } else {
        asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
        if (r.mode >= 2u) store_peers_u32(p, v, r);
    }
}
// K1's two result words of group g, routed
__device__ __forceinline__ void store_vote_result(int32_t *win, uint32_t *meta, int64_t g, int32_t w, uint32_t m, const OutRoute &r) {
    if (r.mode == 4u) {  // full result locally + the wire word in this rank's slot (a push kernel replicates the slot)
        store_local_u32(win + g, (uint32_t)w);
        store_local_u32(meta + g, m);
        const uint32_t support = (m >> 6) & 0x7Fu, present = (m >> 20) & 0x7Fu;
        if (r.wire_wide) {
            if (support != 0 && (uint32_t)w >= (1u << 18)) atomicOr(r.overflow, 1u);
            const uint32_t word = ((uint32_t)w & 0x3FFFFu) | (support << 18) | (present << 25);
            store_local_u32(r.packed + g, word);
            if (r.n_peers) store_peers_u32(r.packed + g, word, r);
        } else {
            if (support > 31u || present > 31u || (support != 0 && (uint32_t)w > 63u)) atomicOr(r.overflow, 1u);
            const uint16_t word = (uint16_t)(((uint32_t)w & 63u) | ((support & 31u) << 6) | ((present & 31u) << 11));
            uint16_t *p = reinterpret_cast<uint16_t *>(r.packed) + g;
            asm volatile("st.global.L1::no_allocate.u16 [%0], %1;" ::"l"(p), "h"(word) : "memory");
            for (int k = 0; k < r.n_peers; ++k)  // fused reassembly: a warp's 32 words are one 64-byte store per peer
                asm volatile("st.global.u16 [%0], %1;" ::"l"(reinterpret_cast<char *>(p) + r.delta[k]), "h"(word) : "memory");
        }
        return;
    }
    if (r.mode != 3u) {
        store_out_u32(win + g, (uint32_t)w, r);
        store_out_u32(meta + g, m, r);
        return;
    }
    store_local_u32(win + g, (uint32_t)w);
    store_local_u32(meta + g, m);
    const uint32_t support = (m >> 6) & 0x7Fu, present = (m >> 20) & 0x7Fu;
    if (support != 0 && (uint32_t)w >= (1u << 18)) atomicOr(r.overflow, 1u);
    const uint32_t word = ((uint32_t)w & 0x3FFFFu) | (support << 18) | (present << 25);
    store_local_u32(r.packed + g, word);
    store_peers_u32(r.packed + g, word, r);
}

__device__ __forceinline__ void store_out_f64(void *p, double v, const OutRoute &r) {
    if (r.mode == 1u) {
        asm volatile("multimem.st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
    } else {
        asm volatile("st.global.L1::no_allocate.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
        if (r.mode >= 2u) store_peers_f64(p, v, r);
    }
}

}  // namespace kc
