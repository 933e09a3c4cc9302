// kllms_b200.cu — C ABI (include/kllms_b200.h) and launchers of the sm_90a (H100) consensus kernels.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
//        (see k_llms_b200/csrc/Makefile; __graft_entry__.build() runs it).
// No torch, no libraries beyond the CUDA runtime; the driver entry point cuTensorMapEncodeTiled is fetched
// through cudaGetDriverEntryPoint so libcuda is not a link-time dependency.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <type_traits>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "../../include/kllms_b200.h"
#include "kc_internal.h"
#include "kc_alignsim.cuh"
#include "kc_common.cuh"
#include "kc_extra.cuh"
#include "kc_medoid.cuh"
#include "kc_numeric.cuh"
#include "kc_numeric_medoid.cuh"
#include "kc_push.cuh"
#include "kc_vote.cuh"

namespace {
thread_local char g_err[512] = "";
}  // namespace

int kc_fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

namespace {

struct DeviceInfo {
    int sm_count = 0;
    int cc_major = 0;
};

int device_info(DeviceInfo &info) {
    int dev = 0;
    KC_CUDA_I(cudaGetDevice(&dev));
    static std::mutex mu;
    static std::vector<DeviceInfo> cache;
    std::lock_guard<std::mutex> lock(mu);
    if ((int)cache.size() <= dev) cache.resize(dev + 1);
    if (cache[dev].sm_count == 0) {
        KC_CUDA_I(cudaDeviceGetAttribute(&cache[dev].sm_count, cudaDevAttrMultiProcessorCount, dev));
        KC_CUDA_I(cudaDeviceGetAttribute(&cache[dev].cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    }
    info = cache[dev];
    if (info.cc_major != 9) return kc_fail(KC_ENODEV, "device %d has compute capability %d.x; this library is sm_90a only", dev, info.cc_major);
    return KC_OK;
}

// grid of a grid-stride kernel: one CTA per block of work, at most 8 per SM
int stride_grid(int64_t blocks, int &grid) {
    DeviceInfo info;
    int rc = device_info(info);
    if (rc) return rc;
    grid = (int)std::min<int64_t>(blocks, (int64_t)info.sm_count * 8);
    return KC_OK;
}

// grid of a kernel sized by its occupancy: one CTA per block of work, at most one wave of resident CTAs
template <typename Kernel>
int persistent_grid(Kernel kernel, int threads, size_t smem, int64_t blocks, int &grid) {
    DeviceInfo info;
    int rc = device_info(info);
    if (rc) return rc;
    KC_CUDA_I(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    KC_CUDA_I(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
    if (per_sm < 1) return kc_fail(KC_ECUDA, "kernel does not fit on an SM (%d threads, smem %zu)", threads, smem);
    grid = (int)std::min<int64_t>(blocks, (int64_t)info.sm_count * per_sm);
    return KC_OK;
}

// f(std::integral_constant<int, NP>{}) for NP = n rounded up to a power of two, at least NP0 and at most KC_MAX_CANDIDATES
template <int NP0, typename F>
int with_pow2(int n, F &&f) {
    if constexpr (NP0 < KC_MAX_CANDIDATES) {
        if (n > NP0) return with_pow2<NP0 * 2>(n, f);
    }
    return f(std::integral_constant<int, NP0>{});
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---------------------------------------------------------------- TMA descriptor

using EncodeTiledFn = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                   const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int get_encode_fn(EncodeTiledFn &fn) {
    static EncodeTiledFn cached = nullptr;
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (!cached) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        KC_CUDA_I(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        if (q != cudaDriverEntryPointSuccess || !p) return kc_fail(KC_ECUDA, "cuTensorMapEncodeTiled entry point unavailable");
        cached = reinterpret_cast<EncodeTiledFn>(p);
    }
    fn = cached;
    return KC_OK;
}

// rows of `row_bytes` (a power of two in [32, 512]) viewed as a 2-D int32 tensor whose inner extent is
// min(row_bytes, 128) bytes — the widest span a TMA swizzle mode covers; box = TILE groups.
int make_row_tensor_map(CUtensorMap &map, const void *base, int64_t n_groups, int row_bytes, int tile_groups) {
    EncodeTiledFn encode = nullptr;
    int rc = get_encode_fn(encode);
    if (rc) return rc;
    const int inner_bytes = std::min(row_bytes, 128);
    const int rows_per_group = row_bytes / inner_bytes;
    cuuint64_t dims[2] = {(cuuint64_t)(inner_bytes / 4), (cuuint64_t)n_groups * rows_per_group};
    cuuint64_t strides[1] = {(cuuint64_t)inner_bytes};
    cuuint32_t box[2] = {(cuuint32_t)(inner_bytes / 4), (cuuint32_t)(tile_groups * rows_per_group)};
    cuuint32_t elem_strides[2] = {1, 1};
    const CUtensorMapSwizzle swz = inner_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : inner_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                       : CU_TENSOR_MAP_SWIZZLE_32B;
    CUresult r = encode(&map, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<void *>(base), dims, strides, box, elem_strides,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return kc_fail(KC_ECUDA, "cuTensorMapEncodeTiled failed: CUresult %d", (int)r);
    return KC_OK;
}

// A TMA tile coordinate is int32: launch in slabs of at most this many groups.
constexpr int64_t kMaxGroupsPerLaunch = (int64_t)1 << 28;

// A TMA front-end over G rows of `row_bytes`: tiles of 32 rows, one warp per tile, one wave of resident CTAs, in slabs of
// at most kMaxGroupsPerLaunch rows.  A slab is a whole number of `rows_per_record` rows, so that
// (g - g0) % n_fields == g % n_fields.  launch(grid, map, g0, gs) launches `kernel` on rows [g0, g0 + gs).
template <typename Kernel, typename Launch>
int launch_tma_slabs(Kernel kernel, int warps, size_t smem, const void *rows, int64_t G, int row_bytes, int64_t rows_per_record,
                     Launch &&launch) {
    const int64_t slab = std::max<int64_t>(rows_per_record, kMaxGroupsPerLaunch / rows_per_record * rows_per_record);
    for (int64_t g0 = 0; g0 < G; g0 += slab) {
        const int64_t gs = std::min(slab, G - g0);
        CUtensorMap map;
        int rc = make_row_tensor_map(map, static_cast<const char *>(rows) + g0 * row_bytes, gs, row_bytes, 32);
        if (rc) return rc;
        int grid = 0;
        rc = persistent_grid(kernel, warps * 32, smem, ((gs + 31) / 32 + warps - 1) / warps, grid);
        if (rc) return rc;
        launch(grid, map, g0, gs);
        KC_CUDA_I(cudaGetLastError());
    }
    return KC_OK;
}

// K3b's weight rows: `wrow` floats per record in stream-ordered scratch on st, written by pre(grid, rows) (a weight_rows
// kernel, 8 records per 256-thread CTA) and read by vote(rows); the scratch is freed on st on every path.  Without records
// there are no rows: vote(nullptr).
template <typename Pre, typename Vote>
int with_weight_rows(int64_t n_records, int wrow, cudaStream_t st, const char *who, Pre &&pre, Vote &&vote) {
    if (n_records == 0) return vote(nullptr);
    int grid = 0;
    int rc = stride_grid((n_records + 7) / 8, grid);
    if (rc) return rc;
    float *rows = nullptr;
    KC_CUDA_I(cudaMallocAsync(reinterpret_cast<void **>(&rows), (size_t)n_records * wrow * 4, st));
    pre(grid, rows);
    rc = cudaGetLastError() == cudaSuccess ? KC_OK : kc_fail(KC_ECUDA, "%s: weight_rows_kernel launch failed", who);
    if (!rc) rc = vote(rows);
    cudaFreeAsync(rows, st);
    return rc;
}

// ---------------------------------------------------------------- K1 launchers

// The argument checks of K1's entry points, `who` naming the entry in the messages.  Zero groups pass once n is valid:
// there is nothing to launch and the buffers are not looked at.  Without a none_code table every group is field 0.
int check_vote_args(const char *who, const void *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t &n_fields,
                    const void *d_win_code, const void *d_meta) {
    if (n < 1 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "%s: n=%d outside [1,%d]", who, n, KC_MAX_CANDIDATES);
    if (n_groups < 0) return kc_fail(KC_EINVAL, "%s: negative n_groups", who);
    if (n_groups == 0) return KC_OK;
    if (!d_codes || !d_win_code || !d_meta) return kc_fail(KC_EINVAL, "%s: NULL buffer", who);
    if (d_none_code && n_fields < 1) return kc_fail(KC_EINVAL, "%s: none_code given but n_fields=%d", who, n_fields);
    if (!d_none_code) n_fields = 1;
    if (!aligned16(d_codes)) return kc_fail(KC_EINVAL, "%s: d_codes must be 16-byte aligned", who);
    return KC_OK;
}

kc::FieldMap make_field_map(const int32_t *none_code, int n_fields) {
    kc::FieldMap fm;
    fm.none_code = none_code;
    fm.n_fields = (uint32_t)std::max(n_fields, 1);
    fm.magic = (uint32_t)(((uint64_t)1 << 32) / fm.n_fields + 1);
    return fm;
}

template <int N, int WARPS, int STAGES>
int launch_vote_tma(const int32_t *codes, int64_t G, const int32_t *none_code, int n_fields, int32_t *win, uint32_t *meta,
                    cudaStream_t st, kc::OutRoute mc) {
    if (none_code && n_fields >= 60000) return kc_fail(KC_EINVAL, "kc_vote_i32: more than 60000 fields with none_code is not supported");
    const size_t smem = kc::WarpTiles<N * 4, WARPS, STAGES>::RING_BYTES;
    const kc::FieldMap fm = make_field_map(none_code, n_fields);
    auto go = [&](auto kernel) {
        return launch_tma_slabs(kernel, WARPS, smem, codes, G, N * 4, n_fields, [&](int grid, const CUtensorMap &map, int64_t g0, int64_t gs) {
            kernel<<<grid, WARPS * 32, smem, st>>>(map, (uint32_t)gs, fm, win + g0, meta + g0, mc);
        });
    };
    return none_code ? go(kc::vote_tma_kernel<N, WARPS, STAGES, true>) : go(kc::vote_tma_kernel<N, WARPS, STAGES, false>);
}

// Cell: int32_t or int8_t cells.  VEC: n == NP, whole rows; int32 rows from NP = 4 to 16 request the next row before working
// on this one
template <int NP, bool VEC, typename Cell>
int launch_vote_direct(const Cell *codes, int64_t G, int n, const int32_t *none_code, int n_fields, int32_t *win,
                       uint32_t *meta, cudaStream_t st, kc::OutRoute mc) {
    constexpr bool kPrefetch = std::is_same_v<Cell, int32_t> && VEC && NP >= 4 && NP <= 16;
    const int threads = 256;
    int grid = 0;
    int rc = stride_grid((G + threads - 1) / threads, grid);
    if (rc) return rc;
    auto kernel = none_code ? kc::vote_direct_kernel<Cell, NP, VEC, true, kPrefetch> : kc::vote_direct_kernel<Cell, NP, VEC, false, kPrefetch>;
    kernel<<<grid, threads, 0, st>>>(codes, G, n, make_field_map(none_code, n_fields), win, meta, mc);
    KC_CUDA_I(cudaGetLastError());
    return KC_OK;
}

// small rows, local results: GPT consecutive groups per thread (kc::vote_multi_kernel); the remainder (< GPT groups) goes
// through the one-group-per-thread kernel
template <int NP>
int launch_vote_multi(const int32_t *codes, int64_t G, const int32_t *none_code, int n_fields, int32_t *win, uint32_t *meta,
                      cudaStream_t st) {
    constexpr int GPT = 16 / NP;
    const int64_t units = G / GPT;
    if (units > 0) {
        const int threads = 256;
        int grid = 0;
        int rc = stride_grid((units + threads - 1) / threads, grid);
        if (rc) return rc;
        auto kernel = none_code ? kc::vote_multi_kernel<NP, GPT, true> : kc::vote_multi_kernel<NP, GPT, false>;
        kernel<<<grid, threads, 0, st>>>(codes, units, make_field_map(none_code, n_fields), win, meta);
        KC_CUDA_I(cudaGetLastError());
    }
    const int64_t done = units * GPT;
    if (done < G) {  // the last few groups: their field phase continues where the units stopped
        kc::OutRoute local{};
        if (!none_code) return launch_vote_direct<NP, true>(codes + done * NP, G - done, NP, nullptr, 1, win + done, meta + done, st, local);
        // rotate the field table so that group `done` sees its own field first: simplest is one group per launch (< GPT of them)
        for (int64_t g = done; g < G; ++g) {
            const int f = (int)(g % n_fields);
            int rc = launch_vote_direct<NP, true>(codes + g * NP, 1, NP, none_code + f, 1, win + g, meta + g, st, local);
            if (rc) return rc;
        }
    }
    return KC_OK;
}

// ---------------------------------------------------------------- K2 launchers

// FAST: the fast path in front (kc::numeric_tma_fast_kernel), local results only; it re-reads its queue's overflow from `vals`
template <int N, int WARPS, int STAGES, int MIN_CTAS, bool FAST = false>
int launch_numeric_tma(const double *vals, int64_t G, double rel_eps, double abs_eps, double *value, uint32_t *meta,
                       cudaStream_t st, kc::OutRoute mc) {
    constexpr size_t smem = kc::numeric_tma_smem<N, WARPS, STAGES>();
    auto go = [&](auto kernel) {
        return launch_tma_slabs(kernel, WARPS, smem, vals, G, N * 8, 1, [&](int grid, const CUtensorMap &map, int64_t g0, int64_t gs) {
            if constexpr (FAST)
                kernel<<<grid, WARPS * 32, smem, st>>>(map, vals + g0 * N, (uint32_t)gs, rel_eps, abs_eps, value + g0, meta + g0);
            else
                kernel<<<grid, WARPS * 32, smem, st>>>(map, (uint32_t)gs, rel_eps, abs_eps, value + g0, meta + g0, mc);
        });
    };
    if constexpr (FAST) return go(kc::numeric_tma_fast_kernel<N, WARPS, STAGES, MIN_CTAS>);
    else return go(kc::numeric_tma_kernel<N, WARPS, STAGES, MIN_CTAS>);
}

// FAST: the fast path in front (kc::numeric_direct_fast_kernel; n == NP, local results only).  Otherwise PREFETCH (the next
// row requested before this one is worked on) when n == NP and NP is 4 or 8, the sizes whose n == NP reaches this launcher.
template <int NP, int T, bool FAST = false>
int launch_numeric_direct(const double *vals, int64_t G, int n, double rel_eps, double abs_eps, double *value,
                          uint32_t *meta, cudaStream_t st, kc::OutRoute mc) {
    constexpr size_t smem = kc::numeric_direct_smem<NP, T>();
    auto launch = [&](auto kernel, auto... n_arg) -> int {  // n_arg: n, except for the fast kernel
        int grid = 0;
        int rc = persistent_grid(kernel, T, smem, (G + T - 1) / T, grid);
        if (rc) return rc;
        kernel<<<grid, T, smem, st>>>(vals, G, n_arg..., rel_eps, abs_eps, value, meta, mc);
        KC_CUDA_I(cudaGetLastError());
        return KC_OK;
    };
    if constexpr (FAST) {
        return launch(kc::numeric_direct_fast_kernel<NP, T>);
    } else {
        if constexpr (NP == 4 || NP == 8) {
            if (n == NP) return launch(kc::numeric_direct_kernel<NP, T, true>, n);
        }
        return launch(kc::numeric_direct_kernel<NP, T, false>, n);
    }
}

// the n = 2 and n = 4 case analyses (kc::numeric_pairs_kernel, kc::numeric_quads_kernel): GPT groups per thread; the last
// < GPT groups go through the direct kernel
template <int NP, int GPT, typename Kernel>
int launch_numeric_units(Kernel kernel, const double *vals, int64_t G, double rel_eps, double abs_eps, double *value, uint32_t *meta,
                         cudaStream_t st, kc::OutRoute mc) {
    const int64_t units = G / GPT;
    if (units > 0) {
        int grid = 0;
        int rc = stride_grid((units + 255) / 256, grid);
        if (rc) return rc;
        kernel<<<grid, 256, 0, st>>>(vals, units, rel_eps, abs_eps, value, meta);
        KC_CUDA_I(cudaGetLastError());
    }
    const int64_t done = units * GPT;
    if (done == G) return KC_OK;
    return launch_numeric_direct<NP, 128>(vals + done * NP, G - done, NP, rel_eps, abs_eps, value + done, meta + done, st, mc);
}

// Never launched (n = 4 and 8 take other K2 kernels).  The K2 kernels share __noinline__ helpers with these two
// instantiations, and without them compile to different SASS: numeric_tma_fast_kernel<16, 4, 1, 6> spills 12 bytes and
// numeric_tma_kernel<32, 4, 1, 4> needs 127 registers instead of 113 (DESIGN §6).
[[maybe_unused]] void *const kPinNumericSass[] = {(void *)kc::numeric_tma_kernel<4, 8, 2, 3>, (void *)kc::numeric_tma_kernel<8, 8, 2, 3>};
}  // namespace

// ---------------------------------------------------------------- host-buffer context

namespace {
struct HostCtx {
    static constexpr int kStreams = 3;
    int device = -1;
    cudaStream_t streams[kStreams] = {};
    kc::GrowBuf<kc::Mem::Device> codes[kStreams], vals[kStreams], win[kStreams], vmeta[kStreams], value[kStreams], nmeta[kStreams], none;
};
std::mutex g_host_mu;
HostCtx *const g_host = new HostCtx[16];  // never destroyed, like every pooled owner of device memory (kc_internal.h)

}  // namespace

// ================================================================ C ABI

extern "C" {

int kc_version(void) { return KC_VERSION; }

const char *kc_last_error(void) { return g_err; }

int kc_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int ok = 0;
    for (int d = 0; d < n; ++d) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, d) == cudaSuccess && major == 9) ++ok;
    }
    return ok;
}

int kc_sm_count(int device) {
    int sm = 0;
    KC_CUDA_I(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, device));
    return sm;
}

int kc_set_device(int device) {
    KC_CUDA_I(cudaSetDevice(device));
    return KC_OK;
}

int kc_vote_i32(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                int32_t *d_win_code, uint32_t *d_meta, void *stream) {
    return kc_vote_i32_ex(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, KC_OUT_LOCAL, stream);
}

static int make_peer_route(const char *who, int32_t n_peers, const int64_t *peer_delta_bytes, kc::OutRoute &r) {
    if (n_peers < 0 || n_peers > 7) return kc_fail(KC_EINVAL, "%s: n_peers=%d outside [0,7]", who, n_peers);
    if (n_peers > 0 && !peer_delta_bytes) return kc_fail(KC_EINVAL, "%s: NULL peer_delta_bytes", who);
    r = kc::OutRoute{};
    r.mode = KC_OUT_PEERS;
    r.n_peers = n_peers;
    for (int k = 0; k < n_peers; ++k) {
        if (peer_delta_bytes[k] % 8 != 0) return kc_fail(KC_EINVAL, "%s: peer_delta_bytes[%d] is not a multiple of 8", who, k);
        r.delta[k] = (long long)peer_delta_bytes[k];
    }
    return KC_OK;
}

static int vote_i32_routed(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                           int32_t *d_win_code, uint32_t *d_meta, kc::OutRoute mc, void *stream);

int kc_vote_i32_ex(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                   int32_t *d_win_code, uint32_t *d_meta, uint32_t out_mode, void *stream) {
    if (out_mode > KC_OUT_MULTIMEM) return kc_fail(KC_EINVAL, "kc_vote_i32_ex: unknown out_mode %u (peers: kc_vote_i32_peers)", out_mode);
    kc::OutRoute mc{};
    mc.mode = out_mode;
    return vote_i32_routed(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, mc, stream);
}

int kc_vote_i32_peers(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                      int32_t *d_win_code, uint32_t *d_meta, int32_t n_peers, const int64_t *peer_delta_bytes, void *stream) {
    kc::OutRoute mc;
    int rc = make_peer_route("kc_vote_i32_peers", n_peers, peer_delta_bytes, mc);
    if (rc) return rc;
    return vote_i32_routed(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, mc, stream);
}

int kc_vote_i32_peers_packed(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                             int32_t *d_win_code, uint32_t *d_meta, uint32_t *d_packed, int32_t n_peers,
                             const int64_t *peer_delta_bytes, uint32_t *d_overflow, void *stream) {
    if (!d_packed || !d_overflow) return kc_fail(KC_EINVAL, "kc_vote_i32_peers_packed: NULL d_packed / d_overflow");
    kc::OutRoute mc;
    int rc = make_peer_route("kc_vote_i32_peers_packed", n_peers, peer_delta_bytes, mc);
    if (rc) return rc;
    mc.mode = 3u;
    mc.packed = d_packed;
    mc.overflow = d_overflow;
    return vote_i32_routed(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, mc, stream);
}

static int vote_i32_routed(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                           int32_t *d_win_code, uint32_t *d_meta, kc::OutRoute mc, void *stream) {
    const int rc = check_vote_args("kc_vote_i32", d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta);
    if (rc || n_groups == 0) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // measured on H100 SXM (400 W, 1M x 24 fields): the direct front-end wins up to n = 16 (0.59 vs 0.63 ms at n = 16), the
    // TMA pipeline from n = 32 (1.12 vs 1.30 ms at n = 32)
    if (mc.local()) {  // the multi-group kernel only has local stores
        switch (n) {
            case 2: return launch_vote_multi<2>(d_codes, n_groups, d_none_code, n_fields, d_win_code, d_meta, st);
            case 4: return launch_vote_multi<4>(d_codes, n_groups, d_none_code, n_fields, d_win_code, d_meta, st);
            case 8: return launch_vote_multi<8>(d_codes, n_groups, d_none_code, n_fields, d_win_code, d_meta, st);
            default: break;
        }
    }
    switch (n) {
        case 1: return launch_vote_direct<1, true>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        case 2: return launch_vote_direct<2, true>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        case 4: return launch_vote_direct<4, true>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        case 8: return launch_vote_direct<8, true>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        case 16: return launch_vote_direct<16, true>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        case 32: return launch_vote_tma<32, 8, 2>(d_codes, n_groups, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        case 64: return launch_vote_tma<64, 4, 2>(d_codes, n_groups, d_none_code, n_fields, d_win_code, d_meta, st, mc);
        default: break;
    }
    return with_pow2<4>(n, [&](auto np) {
        return launch_vote_direct<decltype(np)::value, false>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, mc);
    });
}

int kc_vote_i32_wire(const int32_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
                     int32_t *d_win_code, uint32_t *d_meta, void *d_wire_words, int32_t wide, int32_t n_peers,
                     const int64_t *peer_delta_bytes, uint32_t *d_overflow, void *stream) {
    if (!d_wire_words || !d_overflow) return kc_fail(KC_EINVAL, "kc_vote_i32_wire: NULL d_wire_words / d_overflow");
    kc::OutRoute mc{};
    if (n_peers) {
        int rc = make_peer_route("kc_vote_i32_wire", n_peers, peer_delta_bytes, mc);
        if (rc) return rc;
    }
    mc.mode = 4u;
    mc.packed = static_cast<uint32_t *>(d_wire_words);
    mc.overflow = d_overflow;
    mc.wire_wide = wide ? 1u : 0u;
    return vote_i32_routed(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, mc, stream);
}

static int fill_push_args(kc::PushArgs &a, const int32_t *d_win_code, const uint32_t *d_vote_meta, int64_t n_vote_groups, const double *d_value,
                          const uint32_t *d_num_meta, int64_t n_num_groups, void *d_wire_votes, void *d_wire_value, void *d_wire_num_meta,
                          int32_t wide, int32_t n_peers, const int64_t *peer_delta_bytes, uint32_t *d_overflow) {
    if (n_vote_groups < 0 || n_num_groups < 0) return kc_fail(KC_EINVAL, "kc_push_results: negative size");
    if (n_vote_groups % 8 || n_num_groups % 8) return kc_fail(KC_EINVAL, "kc_push_results: group counts must be multiples of 8 (whole 16-byte vectors)");
    if (n_peers < 0 || n_peers > 7 || (n_peers && !peer_delta_bytes)) return kc_fail(KC_EINVAL, "kc_push_results: n_peers=%d outside [0,7] or NULL deltas", n_peers);
    if ((n_vote_groups && (((!d_win_code) != (!d_vote_meta)) || !d_wire_votes)) || (n_num_groups && (!d_value || !d_num_meta || !d_wire_value || !d_wire_num_meta)))
        return kc_fail(KC_EINVAL, "kc_push_results: NULL buffer");
    for (const void *p : {(const void *)d_win_code, (const void *)d_vote_meta, (const void *)d_value, (const void *)d_num_meta,
                          (const void *)d_wire_votes, (const void *)d_wire_value, (const void *)d_wire_num_meta})
        if (!aligned16(p)) return kc_fail(KC_EINVAL, "kc_push_results: buffers must be 16-byte aligned");
    a = kc::PushArgs{};
    a.win = d_win_code;
    a.vmeta = d_vote_meta;
    a.gv = n_vote_groups;
    a.value = d_value;
    a.nmeta = d_num_meta;
    a.gx = n_num_groups;
    a.wire_votes = static_cast<uint8_t *>(d_wire_votes);
    a.wire_value = static_cast<uint8_t *>(d_wire_value);
    a.wire_nmeta = static_cast<uint8_t *>(d_wire_num_meta);
    a.n_peers = n_peers;
    for (int k = 0; k < n_peers; ++k) {
        if (peer_delta_bytes[k] % 16 != 0) return kc_fail(KC_EINVAL, "kc_push_results: peer_delta_bytes[%d] is not a multiple of 16", k);
        a.delta[k] = (long long)peer_delta_bytes[k];
    }
    a.wide = wide ? 1 : 0;
    a.overflow = d_overflow;
    return KC_OK;
}

int kc_push_results(const int32_t *d_win_code, const uint32_t *d_vote_meta, int64_t n_vote_groups, const double *d_value,
                    const uint32_t *d_num_meta, int64_t n_num_groups, void *d_wire_votes, void *d_wire_value, void *d_wire_num_meta,
                    int32_t wide, int32_t n_peers, const int64_t *peer_delta_bytes, uint32_t *d_overflow, int32_t max_ctas, void *stream) {
    kc::PushArgs a;
    int rc = fill_push_args(a, d_win_code, d_vote_meta, n_vote_groups, d_value, d_num_meta, n_num_groups, d_wire_votes, d_wire_value,
                            d_wire_num_meta, wide, n_peers, peer_delta_bytes, d_overflow);
    if (rc) return rc;
    if (n_vote_groups == 0 && n_num_groups == 0) return KC_OK;
    DeviceInfo info;
    rc = device_info(info);
    if (rc) return rc;
    const int64_t units = n_vote_groups / (wide ? 4 : 8) + n_num_groups / 2 + n_num_groups / (wide ? 4 : 8);
    int64_t grid = (units + 255) / 256;
    grid = std::min<int64_t>(grid, max_ctas > 0 ? max_ctas : info.sm_count * 2);
    kc::push_kernel<<<(int)std::max<int64_t>(grid, 1), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    KC_CUDA_I(cudaGetLastError());
    return KC_OK;
}

int kc_vote_i8(const int8_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_none_code, int32_t n_fields,
               int32_t *d_win_code, uint32_t *d_meta, void *stream) {
    const int rc = check_vote_args("kc_vote_i8", d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta);
    if (rc || n_groups == 0) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const kc::OutRoute local{};
    // n a power of two from 4 on: whole 16-byte rows; any other n: the next power of two, cells beyond n absent
    return with_pow2<4>(n, [&](auto np) {
        constexpr int NP = decltype(np)::value;
        if (n == NP) return launch_vote_direct<NP, true>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, local);
        return launch_vote_direct<NP, false>(d_codes, n_groups, n, d_none_code, n_fields, d_win_code, d_meta, st, local);
    });
}

int kc_numeric_f64(const double *d_vals, int64_t n_groups, int32_t n, double rel_eps, double abs_eps, double *d_value,
                   uint32_t *d_meta, void *stream) {
    return kc_numeric_f64_ex(d_vals, n_groups, n, rel_eps, abs_eps, d_value, d_meta, KC_OUT_LOCAL, stream);
}

static int numeric_f64_routed(const double *d_vals, int64_t n_groups, int32_t n, double rel_eps, double abs_eps, double *d_value,
                              uint32_t *d_meta, kc::OutRoute mc, void *stream);

int kc_numeric_f64_ex(const double *d_vals, int64_t n_groups, int32_t n, double rel_eps, double abs_eps, double *d_value,
                      uint32_t *d_meta, uint32_t out_mode, void *stream) {
    if (out_mode > KC_OUT_MULTIMEM) return kc_fail(KC_EINVAL, "kc_numeric_f64_ex: unknown out_mode %u (peers: kc_numeric_f64_peers)", out_mode);
    kc::OutRoute mc{};
    mc.mode = out_mode;
    return numeric_f64_routed(d_vals, n_groups, n, rel_eps, abs_eps, d_value, d_meta, mc, stream);
}

int kc_numeric_f64_peers(const double *d_vals, int64_t n_groups, int32_t n, double rel_eps, double abs_eps, double *d_value,
                         uint32_t *d_meta, int32_t n_peers, const int64_t *peer_delta_bytes, void *stream) {
    kc::OutRoute mc;
    int rc = make_peer_route("kc_numeric_f64_peers", n_peers, peer_delta_bytes, mc);
    if (rc) return rc;
    return numeric_f64_routed(d_vals, n_groups, n, rel_eps, abs_eps, d_value, d_meta, mc, stream);
}

static int numeric_f64_routed(const double *d_vals, int64_t n_groups, int32_t n, double rel_eps, double abs_eps, double *d_value,
                              uint32_t *d_meta, kc::OutRoute mc, void *stream) {
    if (n < 1 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "kc_numeric_f64: n=%d outside [1,%d]", n, KC_MAX_CANDIDATES);
    if (n_groups < 0) return kc_fail(KC_EINVAL, "kc_numeric_f64: negative n_groups");
    if (!(rel_eps >= 0.0) || !(abs_eps >= 0.0)) return kc_fail(KC_EINVAL, "kc_numeric_f64: rel_eps/abs_eps must be >= 0");
    if (n_groups == 0) return KC_OK;
    if (!d_vals || !d_value || !d_meta) return kc_fail(KC_EINVAL, "kc_numeric_f64: NULL buffer");
    if (!aligned16(d_vals)) return kc_fail(KC_EINVAL, "kc_numeric_f64: d_vals must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // measured on H100 SXM (400 W, 1M x 8 fields): the TMA pipeline wins from n = 16 (0.43 vs 0.46 ms at n = 16, 0.83 vs
    // 1.03 at n = 32, 2.55 vs 2.78 at n = 64); direct at n <= 8 (tiles too small to prefetch far enough)
    if (mc.local()) {
        // The fast and small-n kernels only have local stores.  The fast kernels store a group's result when it is decided —
        // most lanes at once, the deferred ones later and scattered.  Local stores do not care; multicast stores do (the
        // general kernel's whole-warp stores use the link better than the fast kernel's), and a fused step is NVLink-bound anyway.
        switch (n) {
            case 2: return launch_numeric_units<2, 4>(kc::numeric_pairs_kernel, d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
            case 4: return launch_numeric_units<4, 2>(kc::numeric_quads_kernel, d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
            case 8: return launch_numeric_direct<8, 128, true>(d_vals, n_groups, 8, rel_eps, abs_eps, d_value, d_meta, st, mc);
            case 16: return launch_numeric_tma<16, 4, 1, 6, true>(d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
            case 32: return launch_numeric_tma<32, 4, 1, 4, true>(d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
            default: break;
        }
    }
    switch (n) {
        case 16: return launch_numeric_tma<16, 4, 1, 7>(d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
        case 32: return launch_numeric_tma<32, 4, 1, 4>(d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
        case 64: return launch_numeric_tma<64, 2, 1, 3>(d_vals, n_groups, rel_eps, abs_eps, d_value, d_meta, st, mc);
        default: break;
    }
    return with_pow2<2>(n, [&](auto np) {
        constexpr int NP = decltype(np)::value;
        return launch_numeric_direct<NP, NP == 64 ? 64 : 128>(d_vals, n_groups, n, rel_eps, abs_eps, d_value, d_meta, st, mc);
    });
}

int kc_confidence_f64(const uint32_t *d_meta, int64_t n_groups, int32_t numeric, const double *d_pvf, double *d_conf,
                      void *stream) {
    if (n_groups < 0) return kc_fail(KC_EINVAL, "kc_confidence_f64: negative n_groups");
    if (n_groups == 0) return KC_OK;
    if (!d_meta || !d_conf) return kc_fail(KC_EINVAL, "kc_confidence_f64: NULL buffer");
    const int threads = 256;
    int grid = 0;
    int rc = stride_grid((n_groups + threads - 1) / threads, grid);
    if (rc) return rc;
    kc::confidence_kernel<<<grid, threads, 0, static_cast<cudaStream_t>(stream)>>>(d_meta, n_groups, numeric != 0, d_pvf, d_conf);
    KC_CUDA_I(cudaGetLastError());
    return KC_OK;
}

int kc_logprob_sum_f32(const float *d_logprobs, const int64_t *d_offsets, int64_t n_seq, float *d_sum, void *stream) {
    if (n_seq < 0) return kc_fail(KC_EINVAL, "kc_logprob_sum_f32: negative n_seq");
    if (n_seq == 0) return KC_OK;
    if (!d_offsets || !d_sum) return kc_fail(KC_EINVAL, "kc_logprob_sum_f32: NULL buffer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int grid = 0;
    if (n_seq >= 4096 && aligned16(d_logprobs)) {
        // T sequences per tile, their contiguous tokens staged in shared memory (up to CAP floats; longer tiles fall back to
        // the warp-per-sequence loop inside the kernel).  64 sequences per tile, 24 KB of staged tokens (chosen from
        // {128/48 KB, 64/24 KB, 64/16 KB, 32/12 KB}; 32/12 KB falls back from 96 tokens per sequence on; not re-timed on H100)
        constexpr int T = 64, CAP = 6 * 1024;
        auto kernel = kc::logprob_sum_tile_kernel<T, CAP>;
        const size_t smem = (size_t)(CAP + 4) * sizeof(float);
        int rc = persistent_grid(kernel, T, smem, (n_seq + T - 1) / T, grid);
        if (rc) return rc;
        kernel<<<grid, T, smem, st>>>(d_logprobs, d_offsets, n_seq, d_sum);
    } else {
        int rc = stride_grid((n_seq + 7) / 8, grid);  // 8 warps, one sequence per warp per iteration
        if (rc) return rc;
        kc::logprob_sum_kernel<<<grid, 256, 0, st>>>(d_logprobs, d_offsets, n_seq, d_sum);
    }
    KC_CUDA_I(cudaGetLastError());
    return KC_OK;
}

int kc_weighted_vote_i32(const int32_t *d_codes, const float *d_seq_logprob, int64_t n_records, int32_t n_fields,
                         int32_t n, const int32_t *d_none_code, int32_t *d_win_code, uint32_t *d_meta, float *d_weight,
                         void *stream) {
    if (n < 1 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "kc_weighted_vote_i32: n=%d outside [1,%d]", n, KC_MAX_CANDIDATES);
    if (n_records < 0 || n_fields < 1) return kc_fail(KC_EINVAL, "kc_weighted_vote_i32: bad sizes");
    if (n_records == 0) return KC_OK;
    if (!d_codes || !d_seq_logprob || !d_win_code || !d_meta || !d_weight) return kc_fail(KC_EINVAL, "kc_weighted_vote_i32: NULL buffer");
    const int64_t G = n_records * n_fields;
    const kc::FieldMap fm = make_field_map(d_none_code, n_fields);
    const bool has_nc = d_none_code != nullptr;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((n == 32 || n == 64) && n_fields < 60000) {  // rows through K1's warp-private TMA pipelines
        const int rec_cap = std::min(32, 31 / n_fields + 2);  // records a tile of 32 groups can span
        const uint64_t inv_fields = kc::wv_inv_fields((uint32_t)n_fields);
        // weights: `wrow` floats per record, from `wts`
        auto launch_tma = [&](auto kernel, int N, int warps, size_t smem, const float *wts, int wrow) {
            return launch_tma_slabs(kernel, warps, smem, d_codes, G, N * 4, n_fields, [&](int grid, const CUtensorMap &map, int64_t g0, int64_t gs) {
                kernel<<<grid, warps * 32, smem, st>>>(map, wts + (g0 / n_fields) * wrow, (uint32_t)gs, fm, has_nc, rec_cap, inv_fields,
                                                       d_win_code + g0, d_meta + g0, d_weight + g0);
            });
        };
        if (n == 32 && rec_cap <= 8) {  // weights by a pre-pass, fetched per tile by a bulk copy (n_fields >= 5; n = 32 only)
            constexpr int N = 32, WARPS = 8, STAGES = 2, WROW = kc::kWRowBulk<N>;
            return with_weight_rows(
                n_records, WROW, st, "kc_weighted_vote_i32",
                [&](int grid, float *rows) { kc::weight_rows_kernel<N><<<grid, 256, 0, st>>>(d_seq_logprob, n_records, rows); },
                [&](float *rows) {
                    const size_t smem = kc::weighted_vote_rows_smem<N, WARPS, STAGES>(rec_cap);
                    return launch_tma(kc::weighted_vote_rows_kernel<N, WARPS, STAGES, 3>, N, WARPS, smem, rows, WROW);
                });
        }
        // n = 32 with 3 CTAs / SM (80 registers) and the logprobs requested a tile ahead; n = 64 (2 x the registers per row)
        // without the prefetch (not re-timed on H100)
        if (n == 32)
            return launch_tma(kc::weighted_vote_tma_kernel<32, 8, 2, 3, true>, 32, 8, kc::weighted_vote_tma_smem<32, 8, 2>(rec_cap), d_seq_logprob, 32);
        return launch_tma(kc::weighted_vote_tma_kernel<64, 4, 2, 3, false>, 64, 4, kc::weighted_vote_tma_smem<64, 4, 2>(rec_cap), d_seq_logprob, 64);
    }
    // n < 8: one group per thread, weights computed per group; faster there than the per-record kernel below (H100 SXM,
    // 700 W, 256 K records x 24 fields: 0.07 against 0.16 ms at n = 2, 0.11 against 0.16 ms at n = 4)
    if (n < 8) {
        const int threads = 128;
        int grid = 0;
        int rc = stride_grid((G + threads - 1) / threads, grid);
        if (rc) return rc;
        auto kernel = n <= 2 ? kc::weighted_vote_kernel<2> : n <= 4 ? kc::weighted_vote_kernel<4> : kc::weighted_vote_kernel<8>;
        kernel<<<grid, threads, 0, st>>>(d_codes, d_seq_logprob, G, n, fm, has_nc, d_win_code, d_meta, d_weight);
        KC_CUDA_I(cudaGetLastError());
        return KC_OK;
    }
    // weights once per record, one row per thread straight from global memory
    constexpr int T = 128;
    const int max_recs = T / n_fields + 2;
    return with_pow2<8>(n, [&](auto np) {
        constexpr int NP = decltype(np)::value;
        auto kernel = kc::weighted_vote_rec_kernel<NP, T>;
        const size_t smem = (size_t)max_recs * NP * 4;  // the candidate weights of the tile's records
        int grid = 0;
        int rc = persistent_grid(kernel, T, smem, (G + T - 1) / T, grid);
        if (rc) return rc;
        kernel<<<grid, T, smem, st>>>(d_codes, d_seq_logprob, G, n, fm, has_nc, d_win_code, d_meta, d_weight);
        KC_CUDA_I(cudaGetLastError());
        return KC_OK;
    });
}

int kc_weighted_vote_groups_i8(const int8_t *d_codes, int64_t n_groups, int32_t n, const int32_t *d_group_record,
                               const float *d_seq_logprob, int64_t n_records, int32_t *d_win_code, uint32_t *d_meta, float *d_weight,
                               void *stream) {
    if (n < 1 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "kc_weighted_vote_groups_i8: n=%d outside [1,%d]", n, KC_MAX_CANDIDATES);
    if (n_groups < 0 || n_records < 0) return kc_fail(KC_EINVAL, "kc_weighted_vote_groups_i8: negative sizes");
    if (n_groups == 0) return KC_OK;
    if (!d_codes || !d_group_record || !d_win_code || !d_meta || !d_weight || (n_records > 0 && !d_seq_logprob))
        return kc_fail(KC_EINVAL, "kc_weighted_vote_groups_i8: NULL buffer");
    if (!aligned16(d_codes)) return kc_fail(KC_EINVAL, "kc_weighted_vote_groups_i8: d_codes must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the buckets and row loads of kc_vote_i8: n a power of two from 4 on reads whole rows, any other n the next power of two
    // with the cells beyond n absent
    return with_pow2<4>(n, [&](auto np) -> int {
        constexpr int NP = decltype(np)::value;
        return with_weight_rows(
            n_records, kc::kWRowBulk<NP>, st, "kc_weighted_vote_groups_i8",
            [&](int grid, float *rows) { kc::weight_rows_n_kernel<NP><<<grid, 256, 0, st>>>(d_seq_logprob, n_records, n, rows); },
            [&](float *rows) {
                const int threads = 128;
                int grid = 0;
                int rc = stride_grid((n_groups + threads - 1) / threads, grid);
                if (rc) return rc;
                auto kernel = n == NP ? kc::weighted_vote_groups_kernel<NP, true> : kc::weighted_vote_groups_kernel<NP, false>;
                kernel<<<grid, threads, 0, st>>>(d_codes, n_groups, n, d_group_record, n_records, rows, d_win_code, d_meta, d_weight);
                return cudaGetLastError() == cudaSuccess ? KC_OK : kc_fail(KC_ECUDA, "kc_weighted_vote_groups_i8: launch failed");
            });
    });
}

int kc_medoid_str(const uint8_t *d_chars, const int32_t *d_str_off, const int32_t *d_grp_off, int64_t n_groups,
                  int32_t max_group, int32_t *d_best_idx, double *d_best_avg, void *stream) {
    return kc_medoid_str_method(d_chars, d_str_off, d_grp_off, n_groups, max_group, KC_SIM_LEVENSHTEIN, d_best_idx, d_best_avg, stream);
}

int kc_medoid_str_method(const uint8_t *d_chars, const int32_t *d_str_off, const int32_t *d_grp_off, int64_t n_groups,
                         int32_t max_group, int32_t method, int32_t *d_best_idx, double *d_best_avg, void *stream) {
    if (method < KC_SIM_LEVENSHTEIN || method > KC_SIM_HAMMING) return kc_fail(KC_EINVAL, "kc_medoid_str: unknown similarity method %d", method);
    if (n_groups < 0) return kc_fail(KC_EINVAL, "kc_medoid_str: negative n_groups");
    if (max_group < 2 || max_group > kc::kMedoidMaxN)
        return kc_fail(KC_EINVAL, "kc_medoid_str: max_group=%d outside [2,%d]", max_group, kc::kMedoidMaxN);
    if (n_groups == 0) return KC_OK;
    if (!d_chars || !d_str_off || !d_grp_off || !d_best_idx || !d_best_avg) return kc_fail(KC_EINVAL, "kc_medoid_str: NULL buffer");
    constexpr int WARPS = 4;
    auto kernel = kc::medoid_kernel<WARPS>;
    const size_t per_warp = (kc::MedoidSmem::bytes(max_group) + 15) & ~size_t(15);  // match tables + distances, sized by max_group
    const size_t smem = WARPS * per_warp;
    int grid = 0;
    int rc = persistent_grid(kernel, WARPS * 32, smem, (n_groups + WARPS - 1) / WARPS, grid);
    if (rc) return rc;
    kernel<<<grid, WARPS * 32, smem, static_cast<cudaStream_t>(stream)>>>(d_chars, d_str_off, d_grp_off, n_groups, max_group,
                                                                         d_best_idx, d_best_avg, method);
    KC_CUDA_I(cudaGetLastError());
    return KC_OK;
}

int kc_numeric_medoid_f64(const double *d_cells, int64_t n_groups, int32_t n, int32_t *d_best, double *d_best_avg, void *stream) {
    if (n < 1 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "kc_numeric_medoid_f64: n=%d outside [1,%d]", n, KC_MAX_CANDIDATES);
    if (n_groups < 0) return kc_fail(KC_EINVAL, "kc_numeric_medoid_f64: negative n_groups");
    if (n_groups == 0) return KC_OK;
    if (!d_cells || !d_best || !d_best_avg) return kc_fail(KC_EINVAL, "kc_numeric_medoid_f64: NULL buffer");
    int team = 1;
    while (team < n && team < 32) team *= 2;
    const int64_t groups_per_block = (int64_t)kc::kNumMedoidWarps * (32 / team);
    int grid = 0;
    int rc = stride_grid((n_groups + groups_per_block - 1) / groups_per_block, grid);
    if (rc) return rc;
    kc::numeric_medoid_kernel<<<grid, kc::kNumMedoidWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(d_cells, n_groups, n, team, d_best,
                                                                                                       d_best_avg);
    KC_CUDA_I(cudaGetLastError());
    return KC_OK;
}

int kc_medoid_str_host(const uint8_t *h_chars, int64_t n_chars, const int32_t *h_str_off, const int32_t *h_grp_off, int64_t n_groups,
                       int32_t max_group, int32_t *h_best_idx, double *h_best_avg, int device) {
    if (n_groups < 0 || n_chars < 0) return kc_fail(KC_EINVAL, "kc_medoid_str_host: negative size");
    if (n_groups == 0) return KC_OK;
    if (!h_str_off || !h_grp_off || !h_best_idx || !h_best_avg || (n_chars && !h_chars)) return kc_fail(KC_EINVAL, "kc_medoid_str_host: NULL buffer");
    KC_CUDA_I(cudaSetDevice(device));
    const int64_t n_str = h_grp_off[n_groups];
    if (n_str < 0 || h_str_off[n_str] != n_chars) return kc_fail(KC_EINVAL, "kc_medoid_str_host: offsets do not add up to n_chars");
    kc::Staged st("kc_medoid_str_host");
    uint8_t *d[5];  // chars, str_off, grp_off, best_idx, best_avg
    if (const int rc = st.alloc({(size_t)n_chars + 256, ((size_t)n_str + 1) * 4, ((size_t)n_groups + 1) * 4, (size_t)n_groups * 4, (size_t)n_groups * 8}, d))
        return rc;
    if (n_chars) st.check(cudaMemcpyAsync(d[0], h_chars, (size_t)n_chars, cudaMemcpyHostToDevice, st.stream), "H2D chars");
    st.check(cudaMemcpyAsync(d[1], h_str_off, ((size_t)n_str + 1) * 4, cudaMemcpyHostToDevice, st.stream), "H2D str_off");
    st.check(cudaMemcpyAsync(d[2], h_grp_off, ((size_t)n_groups + 1) * 4, cudaMemcpyHostToDevice, st.stream), "H2D grp_off");
    if (st.rc == KC_OK)
        st.rc = kc_medoid_str(d[0], reinterpret_cast<int32_t *>(d[1]), reinterpret_cast<int32_t *>(d[2]), n_groups, max_group,
                              reinterpret_cast<int32_t *>(d[3]), reinterpret_cast<double *>(d[4]), st.stream);
    st.check(cudaMemcpyAsync(h_best_idx, d[3], (size_t)n_groups * 4, cudaMemcpyDeviceToHost, st.stream), "D2H idx");
    st.check(cudaMemcpyAsync(h_best_avg, d[4], (size_t)n_groups * 8, cudaMemcpyDeviceToHost, st.stream), "D2H avg");
    return st.finish();
}

// Element similarities of the list-alignment pre-pass (kc_alignsim.cuh): H2D of the value table, one launch, D2H of the
// matrices (synchronous); device < 0 runs the same phase on the calling host thread, lane 0 .. host_lanes - 1 of each node in turn.
int kc_alignsim(const KcAsNode *nodes, int64_t n_nodes, const KcAsVal *vals, int64_t n_vals, const uint8_t *chars, int64_t n_chars,
                double *h_out, int64_t n_out, int device, int host_lanes, int64_t *pairs) {
    if (pairs) *pairs = 0;
    if (n_nodes < 0 || n_vals < 0 || n_chars < 0 || n_out < 0) return kc_fail(KC_EINVAL, "kc_alignsim: negative size");
    if (device < 0 && host_lanes < 1) return kc_fail(KC_EINVAL, "kc_alignsim: host_lanes < 1");
    if (n_nodes == 0) return KC_OK;
    if (!nodes || !vals || !h_out || (n_chars && !chars)) return kc_fail(KC_EINVAL, "kc_alignsim: NULL buffer");
    if (device < 0) {
        uint64_t tab[kc::kPeqStride];
        int64_t decided = 0;
        for (int64_t g = 0; g < n_nodes; ++g)
            for (int lane = 0; lane < host_lanes; ++lane) decided += kc::alignsim_node(nodes[g], vals, chars, h_out, lane, host_lanes, tab);
        if (pairs) *pairs = decided;
        return KC_OK;
    }
    KC_CUDA_I(cudaSetDevice(device));
    kc::Staged st("kc_alignsim");
    uint8_t *d[5];  // decided pairs, nodes, values, chars, matrices
    if (const int rc = st.alloc({8, (size_t)n_nodes * sizeof(KcAsNode), (size_t)n_vals * sizeof(KcAsVal), (size_t)n_chars, (size_t)n_out * 8}, d))
        return rc;
    st.check(cudaMemsetAsync(d[0], 0, 8, st.stream), "memset");
    st.check(cudaMemcpyAsync(d[1], nodes, (size_t)n_nodes * sizeof(KcAsNode), cudaMemcpyHostToDevice, st.stream), "H2D nodes");
    if (n_vals) st.check(cudaMemcpyAsync(d[2], vals, (size_t)n_vals * sizeof(KcAsVal), cudaMemcpyHostToDevice, st.stream), "H2D values");
    if (n_chars) st.check(cudaMemcpyAsync(d[3], chars, (size_t)n_chars, cudaMemcpyHostToDevice, st.stream), "H2D chars");
    constexpr int WARPS = 4;
    auto kernel = kc::alignsim_kernel<WARPS>;
    int grid = 0;
    if (st.rc == KC_OK) st.rc = persistent_grid(kernel, WARPS * 32, 0, (n_nodes + WARPS - 1) / WARPS, grid);
    if (st.rc == KC_OK) {
        kernel<<<grid, WARPS * 32, 0, st.stream>>>(reinterpret_cast<const KcAsNode *>(d[1]), n_nodes, reinterpret_cast<const KcAsVal *>(d[2]),
                                                   d[3], reinterpret_cast<double *>(d[4]), reinterpret_cast<unsigned long long *>(d[0]));
        st.check(cudaGetLastError(), "launch");
    }
    unsigned long long decided = 0;
    if (n_out) st.check(cudaMemcpyAsync(h_out, d[4], (size_t)n_out * 8, cudaMemcpyDeviceToHost, st.stream), "D2H matrices");
    st.check(cudaMemcpyAsync(&decided, d[0], 8, cudaMemcpyDeviceToHost, st.stream), "D2H pairs");
    const int rc = st.finish();
    if (pairs) *pairs = (int64_t)decided;
    return rc;
}

void *kc_host_alloc(uint64_t bytes) {
    void *p = nullptr;
    return kc::pinned_alloc(&p, bytes ? bytes : 1, "kc_host_alloc") ? nullptr : p;
}

void kc_host_free(void *p) { kc::pinned_free(p); }

// ---------------------------------------------------------------- end-to-end with host buffers

static int consensus_host_impl(const void *h_codes_v, int code_bytes, int32_t n_vote_fields, const int32_t *h_none_code,
                               const double *h_vals, int32_t n_num_fields, int64_t n_records, int32_t n, double rel_eps,
                               double abs_eps, int32_t *h_win_code, uint32_t *h_vote_meta, double *h_value,
                               uint32_t *h_num_meta, int device, float *device_ms);

int kc_consensus_host(const int32_t *h_codes, int32_t n_vote_fields, const int32_t *h_none_code, const double *h_vals,
                      int32_t n_num_fields, int64_t n_records, int32_t n, double rel_eps, double abs_eps,
                      int32_t *h_win_code, uint32_t *h_vote_meta, double *h_value, uint32_t *h_num_meta, int device,
                      float *device_ms) {
    return consensus_host_impl(h_codes, 4, n_vote_fields, h_none_code, h_vals, n_num_fields, n_records, n, rel_eps, abs_eps,
                               h_win_code, h_vote_meta, h_value, h_num_meta, device, device_ms);
}

int kc_consensus_host_i8(const int8_t *h_codes, int32_t n_vote_fields, const int32_t *h_none_code, const double *h_vals,
                         int32_t n_num_fields, int64_t n_records, int32_t n, double rel_eps, double abs_eps,
                         int32_t *h_win_code, uint32_t *h_vote_meta, double *h_value, uint32_t *h_num_meta, int device,
                         float *device_ms) {
    return consensus_host_impl(h_codes, 1, n_vote_fields, h_none_code, h_vals, n_num_fields, n_records, n, rel_eps, abs_eps,
                               h_win_code, h_vote_meta, h_value, h_num_meta, device, device_ms);
}

static int consensus_host_impl(const void *h_codes_v, int code_bytes, int32_t n_vote_fields, const int32_t *h_none_code,
                               const double *h_vals, int32_t n_num_fields, int64_t n_records, int32_t n, double rel_eps,
                               double abs_eps, int32_t *h_win_code, uint32_t *h_vote_meta, double *h_value,
                               uint32_t *h_num_meta, int device, float *device_ms) {
    const uint8_t *h_codes = static_cast<const uint8_t *>(h_codes_v);
    if (device_ms) *device_ms = 0.0f;
    if (n < 1 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "kc_consensus_host: n=%d outside [1,%d]", n, KC_MAX_CANDIDATES);
    if (n_records < 0 || n_vote_fields < 0 || n_num_fields < 0) return kc_fail(KC_EINVAL, "kc_consensus_host: negative size");
    if (device < 0 || device >= 16) return kc_fail(KC_EINVAL, "kc_consensus_host: device %d out of range", device);
    if (n_vote_fields > 0 && (!h_codes || !h_win_code || !h_vote_meta)) return kc_fail(KC_EINVAL, "kc_consensus_host: NULL vote buffer");
    if (n_num_fields > 0 && (!h_vals || !h_value || !h_num_meta)) return kc_fail(KC_EINVAL, "kc_consensus_host: NULL numeric buffer");
    if (n_records == 0 || (n_vote_fields == 0 && n_num_fields == 0)) return KC_OK;

    std::lock_guard<std::mutex> lock(g_host_mu);
    int prev = 0;
    KC_CUDA_I(cudaGetDevice(&prev));
    KC_CUDA_I(cudaSetDevice(device));
    HostCtx &cx = g_host[device];
    int rc = KC_OK;
    auto finish = [&](int code) {
        cudaSetDevice(prev);
        return code;
    };
    if (cx.device != device) {
        for (auto &s : cx.streams)
            if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) return finish(kc_fail(KC_ECUDA, "cudaStreamCreate failed"));
        cx.device = device;
    }
    // chunk: ~48 MiB of input per stream buffer keeps H2D, kernels and D2H of neighbouring chunks overlapped
    const size_t rec_in = (size_t)n * ((size_t)n_vote_fields * code_bytes + (size_t)n_num_fields * 8);
    int64_t chunk = std::max<int64_t>(1024, (int64_t)((48u << 20) / std::max<size_t>(rec_in, 1)));
    chunk = std::min<int64_t>(chunk, n_records);
    chunk = (chunk + 255) / 256 * 256;
    for (int s = 0; s < HostCtx::kStreams && !rc; ++s) {
        if (n_vote_fields) {
            rc = cx.codes[s].reserve((size_t)chunk * n_vote_fields * n * code_bytes);
            if (!rc) rc = cx.win[s].reserve((size_t)chunk * n_vote_fields * 4);
            if (!rc) rc = cx.vmeta[s].reserve((size_t)chunk * n_vote_fields * 4);
        }
        if (n_num_fields && !rc) {
            rc = cx.vals[s].reserve((size_t)chunk * n_num_fields * n * 8);
            if (!rc) rc = cx.value[s].reserve((size_t)chunk * n_num_fields * 8);
            if (!rc) rc = cx.nmeta[s].reserve((size_t)chunk * n_num_fields * 4);
        }
    }
    if (rc) return finish(rc);
    const int32_t *d_none = nullptr;
    if (h_none_code && n_vote_fields) {
        rc = cx.none.reserve((size_t)n_vote_fields * 4);
        if (rc) return finish(rc);
        if (cudaMemcpyAsync(cx.none.p, h_none_code, (size_t)n_vote_fields * 4, cudaMemcpyHostToDevice, cx.streams[0]) != cudaSuccess ||
            cudaStreamSynchronize(cx.streams[0]) != cudaSuccess)
            return finish(kc_fail(KC_ECUDA, "none_code upload failed: %s", cudaGetErrorString(cudaGetLastError())));
        d_none = cx.none.as<int32_t>();
    }
    // device-side timing of the whole call: start on stream 0 before the first copy; stop on stream 0 after it has
    // waited for the other streams' last work
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_join[HostCtx::kStreams] = {};
    if (device_ms) {
        cudaEventCreate(&ev_start);
        cudaEventCreate(&ev_stop);
        for (auto &e : ev_join) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
        cudaEventRecord(ev_start, cx.streams[0]);
        for (int s = 1; s < HostCtx::kStreams; ++s) cudaStreamWaitEvent(cx.streams[s], ev_start, 0);  // nothing starts earlier
    }
    int64_t r0 = 0;
    for (int it = 0; r0 < n_records && !rc; ++it, r0 += chunk) {
        const int s = it % HostCtx::kStreams;
        cudaStream_t st = cx.streams[s];
        const int64_t nr = std::min(chunk, n_records - r0);
        cudaError_t e = cudaSuccess;
        nvtxRangePushA("kc_consensus_host: chunk (H2D, K1, K2, D2H)");
        if (n_vote_fields) {
            const int64_t G = nr * n_vote_fields;
            e = cudaMemcpyAsync(cx.codes[s].p, h_codes + (size_t)r0 * n_vote_fields * n * code_bytes, (size_t)G * n * code_bytes,
                                cudaMemcpyHostToDevice, st);
            if (e == cudaSuccess) {
                rc = code_bytes == 1
                         ? kc_vote_i8(cx.codes[s].as<int8_t>(), G, n, d_none, n_vote_fields, cx.win[s].as<int32_t>(), cx.vmeta[s].as<uint32_t>(), st)
                         : kc_vote_i32(cx.codes[s].as<int32_t>(), G, n, d_none, n_vote_fields, cx.win[s].as<int32_t>(), cx.vmeta[s].as<uint32_t>(), st);
                if (rc) { nvtxRangePop(); break; }
                e = cudaMemcpyAsync(h_win_code + r0 * n_vote_fields, cx.win[s].as<int32_t>(), (size_t)G * 4, cudaMemcpyDeviceToHost, st);
            }
            if (e == cudaSuccess)
                e = cudaMemcpyAsync(h_vote_meta + r0 * n_vote_fields, cx.vmeta[s].as<uint32_t>(), (size_t)G * 4, cudaMemcpyDeviceToHost, st);
        }
        if (n_num_fields && e == cudaSuccess) {
            const int64_t G = nr * n_num_fields;
            e = cudaMemcpyAsync(cx.vals[s].as<double>(), h_vals + r0 * n_num_fields * n, (size_t)G * n * 8, cudaMemcpyHostToDevice, st);
            if (e == cudaSuccess) {
                rc = kc_numeric_f64(cx.vals[s].as<double>(), G, n, rel_eps, abs_eps, cx.value[s].as<double>(), cx.nmeta[s].as<uint32_t>(), st);
                if (rc) { nvtxRangePop(); break; }
                e = cudaMemcpyAsync(h_value + r0 * n_num_fields, cx.value[s].as<double>(), (size_t)G * 8, cudaMemcpyDeviceToHost, st);
            }
            if (e == cudaSuccess)
                e = cudaMemcpyAsync(h_num_meta + r0 * n_num_fields, cx.nmeta[s].as<uint32_t>(), (size_t)G * 4, cudaMemcpyDeviceToHost, st);
        }
        nvtxRangePop();
        if (e != cudaSuccess) rc = kc_fail(KC_ECUDA, "kc_consensus_host: %s", cudaGetErrorString(e));
    }
    if (device_ms) {
        for (int s = 1; s < HostCtx::kStreams; ++s) {
            cudaEventRecord(ev_join[s], cx.streams[s]);
            cudaStreamWaitEvent(cx.streams[0], ev_join[s], 0);
        }
        cudaEventRecord(ev_stop, cx.streams[0]);
    }
    for (auto &s : cx.streams) {
        cudaError_t e = cudaStreamSynchronize(s);
        if (e != cudaSuccess && !rc) rc = kc_fail(KC_ECUDA, "kc_consensus_host sync: %s", cudaGetErrorString(e));
    }
    if (device_ms) {
        if (!rc) cudaEventElapsedTime(device_ms, ev_start, ev_stop);
        cudaEventDestroy(ev_start);
        cudaEventDestroy(ev_stop);
        for (auto &e : ev_join) cudaEventDestroy(e);
    }
    return finish(rc);
}

}  // extern "C"
