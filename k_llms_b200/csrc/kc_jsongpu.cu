// kc_jsongpu.cu — host side of H1g (kc_jsongpu.cuh): kc_consolidate_json_packed() streams a batch of candidate texts through
// the device JSON path in chunks (H2D -> A0 -> A1 -> K1/K2 -> C0 -> C1 -> D2H, several chunks in flight on their own streams),
// hands the records the device path declined to the host path (kc_consolidate_json), and returns the consensus / likelihoods
// texts as one blob with per-record spans.  Also the kc_debug_jsongpu_* test hooks, which run the SAME phase functions on
// the host so the CPU tests can check the logic against the oracle without a GPU (they are not a product path: the product
// entry needs a device and fails without one).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include <cub/device/device_scan.cuh>
#include <nvtx3/nvToolsExt.h>  // header-only; ranges show up in Nsight Systems / ncu --nvtx, cost nothing otherwise

#include "../../include/kllms_b200.h"
#include "kc_internal.h"
#include "kc_jsongpu.cuh"

namespace {

using kc::js::Chunk;
using kc::js::Tok;

#define R_(call)                              \
    do {                                      \
        if (const int rc_ = (call)) return rc_; \
    } while (0)

// Every array of a chunk that the device worker and the host twin both size, each named once: the Stage that sizes it (OFF:
// the chunk does not use it), its length (a count of one of the Units, times a number per unit, plus a constant), the byte
// its new elements are filled with, and whether the device fills them too (the twin fills every array; the device only what
// is read without having been written: rows of records declined while encoding, counts of records declined before
// slots_phase, entry R of the scanned counts).  alloc(k, ptr, len, keep, fill, on_device) sizes buffer k for len elements
// keeping the first `keep` (the slots A1 wrote, when the union round adds its rows), binds ptr to it and fills the rest.
enum Stage { RECORDS, SLOTS, UNION, SCRATCH, CSR, OFF };  // before A0, after the slot scan and U2, before U1, after U1, before A2
struct Units {  // records and text bytes; then field slots, union-round records and union scratch entries, counted on the device
    size_t R, B, T = 0, P = 0, S = 0;
};
template <class Alloc>
int chunk_arrays(const Alloc &alloc, Chunk &ch, Stage stage, const Units &u, size_t keep, bool vrec) {
    const size_t n = (size_t)ch.n;
    int k = 0;
    auto a = [&](Stage st, auto *&ptr, size_t count, size_t per, size_t plus, int fill, bool on_device) {
        const int i = k++;
        return st == stage ? alloc(i, ptr, count * per + plus, keep * per, fill, on_device) : KC_OK;
    };
    R_(a(RECORDS, ch.fcount, u.R, 1, 1, 0, true));
    R_(a(RECORDS, ch.slot, u.R, 1, 1, 0, false));
    R_(a(RECORDS, ch.status, u.R, 1, 0, 0, false));
    R_(a(RECORDS, ch.nest, u.R, 1, 0, 0, false));
    R_(a(RECORDS, ch.pend, u.R, 1, 0, 0, false));
    R_(a(RECORDS, ch.plist, u.R, 1, 1, 0xFF, false));  // -1
    R_(a(ch.lists ? RECORDS : OFF, ch.lst, u.R, 1, 0, 0, false));
    R_(a(RECORDS, ch.vbase, u.R, 1, 0, 0, false));
    R_(a(RECORDS, ch.xbase, u.R, 1, 0, 0, false));
    R_(a(RECORDS, ch.mcount, u.R, 1, 1, 0, true));
    R_(a(RECORDS, ch.scount, u.R, 1, 1, 0, true));
    R_(a(RECORDS, ch.ccount, u.R, 1, 1, 0, true));
    R_(a(RECORDS, ch.len_c, u.R, 1, 1, 0, true));
    R_(a(RECORDS, ch.len_l, u.R, 1, 1, 0, true));
    R_(a(SLOTS, ch.toks, u.T, n, 1, 0, false));
    R_(a(SLOTS, ch.fdesc, u.T, 1, 1, 0, false));
    R_(a(SLOTS, ch.gpos, u.T, 1, 1, 0, false));
    R_(a(SLOTS, ch.piece_c, u.T, 1, 1, 0, false));
    R_(a(SLOTS, ch.piece_l, u.T, 1, 1, 0, false));
    R_(a(SLOTS, ch.vcells, u.T, n, 16, 0xFF, true));  // KC_CODE_NONE
    R_(a(SLOTS, ch.xcells, u.T, n, 2, 0, true));
    R_(a(vrec ? SLOTS : OFF, ch.vrec, u.T, 1, 1, 0xFF, false));  // -1
    R_(a(UNION, ch.ucand, u.P, n, 0, 0, false));
    R_(a(UNION, ch.ubase, u.P, 1, 0, 0, false));
    R_(a(UNION, ch.usize, u.P, 1, 0, 0, false));
    R_(a(SCRATCH, ch.utok, u.S, 1, 0, 0, false));
    R_(a(SCRATCH, ch.unode, u.S, 1, 0, 0, false));
    R_(a(SCRATCH, ch.umap, u.S, 1, 0, 0xFF, false));  // -1
    // upper bounds (no read-back): normalised characters are a subset of the text, <= n strings a group, <= fcount groups a record
    R_(a(CSR, ch.mchars, u.B, 1, 16, 0, false));
    R_(a(CSR, ch.mstr_off, u.T, n, 2, 0, false));
    R_(a(CSR, ch.mgrp_off, u.T, 1, 2, 0, false));
    return KC_OK;
}

// the Chunk's switches for a call's flags, in round `lists` (Chunk::lists); records [aligned0, R) are in the aligned round
void set_flags(Chunk &ch, uint32_t flags, uint8_t lists, int32_t aligned0) {
    ch.xmedoid = (flags & KC_JSON_NUMERIC_MEDOID) != 0;
    ch.key_union = (flags & KC_JSON_KEY_UNION) != 0;
    ch.unicode = (flags & KC_JSON_UNICODE) != 0;
    ch.lists = lists;
    ch.aligned0 = aligned0;
}

// Everything one in-flight chunk needs on the device.  Workers are pooled per device and reused across calls.
struct Worker {
    int device = -1;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[7] = {};
    kc::GrowBuf<kc::Mem::Device> text, off, counters, win, vmeta, xvalue, xmeta, out_c, out_l, scan_tmp, midx, mavg, seq, vweight;
    std::vector<kc::GrowBuf<kc::Mem::Device>> arrays;  // chunk_arrays
    kc::GrowBuf<kc::Mem::Pinned> h_small;  // totals and counters (pinned so the small D2H copies are asynchronous)
    kc::GrowBuf<kc::Mem::Pinned> h_scan;   // the scanned record offsets and the statuses of a chunk
    bool busy = false;
    int init(int dev) {
        if (device == dev) return KC_OK;
        KC_CUDA_I(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        for (auto &e : ev) KC_CUDA_I(cudaEventCreate(&e));
        device = dev;
        return KC_OK;
    }
};

std::mutex g_pool_mu;
std::vector<Worker *> g_workers;  // never freed: device buffers live as long as the process

Worker *acquire_worker(int device) {
    std::lock_guard<std::mutex> lock(g_pool_mu);
    for (Worker *w : g_workers)
        if (!w->busy && w->device == device) {
            w->busy = true;
            return w;
        }
    Worker *w = new Worker;
    w->busy = true;
    g_workers.push_back(w);
    return w;
}
void release_worker(Worker *w) {
    std::lock_guard<std::mutex> lock(g_pool_mu);
    w->busy = false;
}

// pinned output blobs are expensive to create (page-locking): recycle them across calls
struct PinnedBlob {
    char *p = nullptr;
    size_t cap = 0;
};
std::vector<PinnedBlob> g_blob_pool;

PinnedBlob acquire_blob(size_t need) {
    {
        std::lock_guard<std::mutex> lock(g_pool_mu);
        int best = -1;
        for (int i = 0; i < (int)g_blob_pool.size(); ++i)
            if (g_blob_pool[i].cap >= need && (best < 0 || g_blob_pool[i].cap < g_blob_pool[best].cap)) best = i;
        if (best >= 0) {
            PinnedBlob b = g_blob_pool[best];
            g_blob_pool.erase(g_blob_pool.begin() + best);
            return b;
        }
    }
    void *p = nullptr;
    if (kc::pinned_alloc(&p, need, "kc_consolidate_json_packed")) return PinnedBlob{};
    return PinnedBlob{(char *)p, need};
}
void release_blob(PinnedBlob b) {
    if (!b.p) return;
    std::lock_guard<std::mutex> lock(g_pool_mu);
    // small blobs (single requests, many callers at once) are cheap to keep: up to 64 of them; of the large ones the largest four
    size_t n_small = 0, n_large = 0;
    for (auto &x : g_blob_pool) (x.cap <= ((size_t)4 << 20) ? n_small : n_large)++;
    if (b.cap <= ((size_t)4 << 20) && n_small < 64) {
        g_blob_pool.push_back(b);
        return;
    }
    if (n_large >= 4 || b.cap <= ((size_t)4 << 20)) {
        int smallest = -1;
        for (int i = 0; i < (int)g_blob_pool.size(); ++i)
            if (g_blob_pool[i].cap > ((size_t)4 << 20) && (smallest < 0 || g_blob_pool[i].cap < g_blob_pool[smallest].cap)) smallest = i;
        if (smallest < 0 || g_blob_pool[smallest].cap >= b.cap) {
            kc::pinned_free(b.p);
            return;
        }
        kc::pinned_free(g_blob_pool[smallest].p);
        g_blob_pool.erase(g_blob_pool.begin() + smallest);
    }
    g_blob_pool.push_back(b);
}

int team_size(int n) {
    int t = 2;
    while (t < n && t < 32) t *= 2;
    return t;
}

// the chunk arrays of one stage in the worker's device buffers (grown and filled on its stream), and with the slots the result
// arrays of K1 (or K3b), K2 (or K5) beside them
int device_arrays(Worker &w, Chunk &ch, Stage stage, const Units &u, size_t keep, bool weighted) {
    auto dev = [&](int k, auto *&ptr, size_t len, size_t keep_len, int fill, bool on_device) -> int {
        using E = std::remove_reference_t<decltype(*ptr)>;
        if (w.arrays.size() <= (size_t)k) w.arrays.resize((size_t)k + 1);
        R_(w.arrays[(size_t)k].grow(len * sizeof(E), keep_len * sizeof(E), w.stream));
        ptr = w.arrays[(size_t)k].as<E>();
        if (on_device) KC_CUDA_I(cudaMemsetAsync(ptr + keep_len, fill, (len - keep_len) * sizeof(E), w.stream));
        return KC_OK;
    };
    R_(chunk_arrays(dev, ch, stage, u, keep, weighted));
    if (stage != SLOTS) return KC_OK;
    const size_t T1 = std::max<size_t>(u.T, 1);
    R_(w.win.reserve(T1 * 4));
    R_(w.vmeta.reserve(T1 * 4));
    R_(w.xvalue.reserve(T1 * 8));
    R_(w.xmeta.reserve(T1 * 4));
    ch.vmeta = w.vmeta.as<uint32_t>();
    ch.xvalue = w.xvalue.as<double>();
    ch.xmeta = w.xmeta.as<uint32_t>();
    ch.xbest = w.xmeta.as<int32_t>();  // K5 writes its results where K2 would
    ch.xavg = w.xvalue.as<double>();
    if (weighted) {
        R_(w.vweight.reserve(T1 * 4));
        ch.vweight = w.vweight.as<float>();
    }
    return KC_OK;
}

template <typename T>
void exclusive_scan(T *v, size_t len) {  // in place, as cub::DeviceScan::ExclusiveSum
    T acc = 0;
    for (size_t i = 0; i < len; ++i) {
        const T c = v[i];
        v[i] = acc;
        acc += c;
    }
}

}  // namespace

struct kc_json_result {
    int64_t R = 0;
    PinnedBlob blob;                   // GPU-written texts (and host-path texts while they fit)
    std::atomic<int64_t> used{0};
    std::vector<int64_t> c_off, c_len, l_off, l_len;
    std::vector<uint8_t> status, why;
    std::string heap;                  // rare: the texts when the host path's share did not fit the pinned blob
    kc_json_stats stats{};
};

namespace {

struct ChunkStage {  // per-chunk device-time split (CUDA events on the chunk's stream)
    float h2d = 0, plan = 0, kernels = 0, emit = 0, d2h = 0;
};

// The union round of a chunk whose A1 sent P records to it (kc_jsongpu.cuh, U1-U3): U1 counts the candidates' tokens and
// reserves scratch, U2 builds the union trees and reserves union rows behind the first round's T slots, U3 writes the tables
// and runs A1's phases on them.  Two read-backs size the scratch and the rows; the arrays A1 has already written grow with
// their contents kept.  On return u.T counts the union rows too, and h_cnt[0..2] the chunk's groups.
int union_round(Worker &w, Chunk &ch, Units &u, int team, int grid, bool weighted, unsigned long long *h_cnt) {
    cudaStream_t s = w.stream;
    const int32_t P = (int32_t)u.P;
    R_(device_arrays(w, ch, UNION, u, 0, weighted));
    ch.uslot = (uint32_t)u.T;
    kc::js::union_count_kernel<<<grid, 128, 0, s>>>(ch, team, P);
    KC_CUDA_I(cudaGetLastError());
    KC_CUDA_I(cudaMemcpyAsync(h_cnt, ch.counters, 48, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaStreamSynchronize(s));
    u.S = std::max<size_t>(h_cnt[4], 1);  // scratch entries: tokens of the candidates, plus a root per record
    if (u.S >= ((size_t)1 << 32)) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: %zu union scratch entries in one chunk", u.S);
    R_(device_arrays(w, ch, SCRATCH, u, 0, weighted));
    kc::js::union_build_kernel<<<grid, 128, 0, s>>>(ch, team, P);
    KC_CUDA_I(cudaGetLastError());
    KC_CUDA_I(cudaMemcpyAsync(h_cnt, ch.counters, 48, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaStreamSynchronize(s));
    if (const size_t U = h_cnt[5]) {
        const size_t keep = u.T;
        u.T += U;
        if (u.T >= ((size_t)1 << 32)) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: %zu field slots in one chunk", u.T);
        R_(device_arrays(w, ch, SLOTS, u, keep, weighted));
    }
    kc::js::union_plan_kernel<<<grid, 128, 0, s>>>(ch, team, P);
    KC_CUDA_I(cudaGetLastError());
    KC_CUDA_I(cudaMemcpyAsync(h_cnt, ch.counters, 48, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaStreamSynchronize(s));
    return KC_OK;
}

// One chunk on one worker: records [r0, r1) of the batch.  h_seq (NULL: count votes): the batch's candidate sums [R][n], the
// vote leaves are likelihood-weighted (K3b over ragged records in K1's place).  flags: the call's KC_JSON_* flags (set_flags);
// lists: Chunk::lists.  dst (NULL: the identity): the result index of each record of the batch (the aligned round's batch is
// the list records, in the order of their result indices).
int run_chunk(Worker &w, const char *h_text, const int64_t *h_off, const float *h_seq, uint32_t flags, uint8_t lists, const int64_t *dst,
              int64_t r0, int64_t r1, int32_t n, double rel_eps, double abs_eps, int sm_count, kc_json_result &res, ChunkStage &st) {
    const int64_t Rc = r1 - r0;
    const int64_t b0 = h_off[r0 * n], b1 = h_off[r1 * n];
    const size_t bytes = (size_t)(b1 - b0);
    if (bytes >= ((size_t)1 << 32)) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: chunk of %zu bytes", bytes);
    cudaStream_t s = w.stream;
    const bool weighted = h_seq != nullptr;
    Chunk ch{};
    ch.R = (int32_t)Rc;
    ch.n = n;
    set_flags(ch, flags, lists, INT32_MAX);  // a chunk is in one round: Chunk::lists says which
    Units u{(size_t)Rc, bytes};
    R_(device_arrays(w, ch, RECORDS, u, 0, weighted));
    R_(w.text.reserve(bytes + 16));
    R_(w.off.reserve((size_t)(Rc * n + 1) * 8));
    R_(w.counters.reserve(48));
    R_(w.h_small.reserve(64));  // the slot total, then the six counters
    R_(w.h_scan.reserve((size_t)(Rc + 1) * 16 + (size_t)Rc));
    if (h_seq) R_(w.seq.reserve((size_t)std::max<int64_t>(Rc * n, 1) * 4));
    size_t tmp_bytes = 0, tmp_bytes32 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (const int64_t *)nullptr, (int64_t *)nullptr, (int)(Rc + 1), s);
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes32, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(Rc + 1), s);
    R_(w.scan_tmp.reserve(std::max(tmp_bytes, tmp_bytes32) + 256));
    ch.text = w.text.as<uint8_t>();
    ch.off = w.off.as<int64_t>();
    ch.counters = w.counters.as<unsigned long long>();

    nvtxRangePushA("kc_json: H2D texts");
    KC_CUDA_I(cudaEventRecord(w.ev[0], s));
    KC_CUDA_I(cudaMemcpyAsync(w.text.p, h_text + b0, bytes, cudaMemcpyHostToDevice, s));
    KC_CUDA_I(cudaMemcpyAsync(w.off.p, h_off + r0 * n, (size_t)(Rc * n + 1) * 8, cudaMemcpyHostToDevice, s));
    if (h_seq) KC_CUDA_I(cudaMemcpyAsync(w.seq.p, h_seq + r0 * n, (size_t)(Rc * n) * 4, cudaMemcpyHostToDevice, s));  // the chunk's sums
    KC_CUDA_I(cudaEventRecord(w.ev[1], s));
    nvtxRangePop();
    nvtxRangePushA("kc_json: plan (A0 count, A1 scan/type/encode)");

    const int team = team_size(n);
    const int tpw = 32 / team;
    auto grid_for = [&](int64_t threads_needed) {
        const int64_t blocks = (threads_needed + 127) / 128;
        return (int)std::max<int64_t>(1, std::min<int64_t>(blocks, (int64_t)sm_count * 16));
    };
    auto team_grid = [&](int64_t units) { return grid_for((units + tpw - 1) / tpw * 32); };  // a warp per tpw units
    // A0: fields per record, then their exclusive scan (entry Rc of fcount is 0, so slot[Rc] is the total)
    kc::js::count_kernel<<<grid_for(Rc), 128, 0, s>>>(ch);
    KC_CUDA_I(cudaGetLastError());
    size_t tb = w.scan_tmp.cap;
    KC_CUDA_I(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, tb, (const uint32_t *)ch.fcount, ch.slot, (int)(Rc + 1), s));
    uint32_t *h_total = w.h_small.as<uint32_t>();
    KC_CUDA_I(cudaMemcpyAsync(h_total, ch.slot + Rc, 4, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaStreamSynchronize(s));
    u.T = *h_total;  // field slots of the chunk (after a union round: its rows too)
    R_(device_arrays(w, ch, SLOTS, u, 0, weighted));
    KC_CUDA_I(cudaMemsetAsync(w.counters.p, 0, 48, s));
    int64_t gv = 0, gx = 0, gm = 0;
    if (u.T) {
        kc::js::plan_kernel<<<team_grid(Rc), 128, 0, s>>>(ch, team);
        KC_CUDA_I(cudaGetLastError());
        unsigned long long *h_cnt = w.h_small.as<unsigned long long>() + 1;
        KC_CUDA_I(cudaMemcpyAsync(h_cnt, w.counters.p, 32, cudaMemcpyDeviceToHost, s));
        KC_CUDA_I(cudaStreamSynchronize(s));
        if ((u.P = h_cnt[3]))  // records whose candidates differ in shape
            R_(union_round(w, ch, u, team, team_grid((int64_t)u.P), weighted, h_cnt));
        gv = (int64_t)h_cnt[0];
        gx = (int64_t)h_cnt[1];
        gm = (int64_t)h_cnt[2];
    }
    if (gm) {
        // A2: multi-word string fields -> K4's CSR input
        R_(device_arrays(w, ch, CSR, u, 0, weighted));
        R_(w.midx.reserve((u.T + 1) * 4));
        R_(w.mavg.reserve((u.T + 1) * 8));
        ch.midx = w.midx.as<int32_t>();
        ch.mavg = w.mavg.as<double>();
        for (uint32_t *cnt : {ch.mcount, ch.scount, ch.ccount}) {
            tb = w.scan_tmp.cap;
            KC_CUDA_I(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, tb, (const uint32_t *)cnt, cnt, (int)(Rc + 1), s));
        }
        kc::js::medoid_kernel<<<team_grid(Rc), 128, 0, s>>>(ch, team);
        KC_CUDA_I(cudaGetLastError());
    }
    KC_CUDA_I(cudaEventRecord(w.ev[2], s));
    nvtxRangePop();
    nvtxRangePushA("kc_json: K1 vote + K2 numeric + K4 medoid");
    // K1 / K2 / K4: the same kernels as the columnar path (one "field" per group: local codes, no none_code table)
    if (gv && h_seq)
        R_(kc_weighted_vote_groups_i8(ch.vcells, gv, n, ch.vrec, w.seq.as<float>(), Rc, w.win.as<int32_t>(), w.vmeta.as<uint32_t>(),
                                      w.vweight.as<float>(), s));
    else if (gv)
        R_(kc_vote_i8(ch.vcells, gv, n, nullptr, 1, w.win.as<int32_t>(), w.vmeta.as<uint32_t>(), s));
    if (gx && ch.xmedoid) R_(kc_numeric_medoid_f64(ch.xcells, gx, n, w.xmeta.as<int32_t>(), w.xvalue.as<double>(), s));
    else if (gx) R_(kc_numeric_f64(ch.xcells, gx, n, rel_eps, abs_eps, w.xvalue.as<double>(), w.xmeta.as<uint32_t>(), s));
    if (gm) R_(kc_medoid_str(ch.mchars, ch.mstr_off, ch.mgrp_off, gm, std::max(2, n), w.midx.as<int32_t>(), w.mavg.as<double>(), s));
    KC_CUDA_I(cudaEventRecord(w.ev[3], s));
    nvtxRangePop();
    nvtxRangePushA("kc_json: emit (C0 lengths, C1 write)");
    // C0: piece lengths and record lengths, then record offsets in the two output blobs
    kc::js::len_kernel<<<team_grid(Rc), 128, 0, s>>>(ch, team);
    KC_CUDA_I(cudaGetLastError());
    tb = w.scan_tmp.cap;
    KC_CUDA_I(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, tb, (const int64_t *)ch.len_c, ch.len_c, (int)(Rc + 1), s));
    tb = w.scan_tmp.cap;
    KC_CUDA_I(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, tb, (const int64_t *)ch.len_l, ch.len_l, (int)(Rc + 1), s));
    int64_t *h_scan_c = w.h_scan.as<int64_t>(), *h_scan_l = h_scan_c + (Rc + 1);
    uint8_t *h_status = (uint8_t *)(h_scan_l + (Rc + 1));
    KC_CUDA_I(cudaMemcpyAsync(h_scan_c, ch.len_c, (size_t)(Rc + 1) * 8, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaMemcpyAsync(h_scan_l, ch.len_l, (size_t)(Rc + 1) * 8, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaMemcpyAsync(h_status, ch.status, (size_t)Rc, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaStreamSynchronize(s));
    const int64_t out_c_bytes = h_scan_c[Rc], out_l_bytes = h_scan_l[Rc];
    R_(w.out_c.reserve((size_t)std::max<int64_t>(out_c_bytes, 1)));
    R_(w.out_l.reserve((size_t)std::max<int64_t>(out_l_bytes, 1)));
    ch.out_c = w.out_c.as<uint8_t>();
    ch.out_l = w.out_l.as<uint8_t>();
    if (out_c_bytes) {
        kc::js::write_kernel<<<team_grid(Rc), 128, 0, s>>>(ch, team);
        KC_CUDA_I(cudaGetLastError());
    }
    KC_CUDA_I(cudaEventRecord(w.ev[4], s));
    nvtxRangePop();
    nvtxRangePushA("kc_json: D2H texts");
    // the chunk's region of the result blob
    const int64_t need = out_c_bytes + out_l_bytes;
    const int64_t pos = res.used.fetch_add(need);
    if (pos + need > (int64_t)res.blob.cap) {  // the estimate of the output size was too small: leave the chunk to the host path
        res.used.fetch_sub(need);
        for (int64_t i = r0; i < r1; ++i) {
            const int64_t r = dst ? dst[i] : i;
            res.status[(size_t)r] = 1;
            res.why[(size_t)r] = (uint8_t)kc::js::D_TOO_LONG;
        }
        return KC_OK;
    }
    if (out_c_bytes) KC_CUDA_I(cudaMemcpyAsync(res.blob.p + pos, ch.out_c, (size_t)out_c_bytes, cudaMemcpyDeviceToHost, s));
    if (out_l_bytes) KC_CUDA_I(cudaMemcpyAsync(res.blob.p + pos + out_c_bytes, ch.out_l, (size_t)out_l_bytes, cudaMemcpyDeviceToHost, s));
    KC_CUDA_I(cudaEventRecord(w.ev[5], s));
    KC_CUDA_I(cudaStreamSynchronize(s));
    nvtxRangePop();
    for (int64_t i = 0; i < Rc; ++i) {
        const int64_t r = dst ? dst[r0 + i] : r0 + i;
        res.status[(size_t)r] = h_status[i] ? 1 : 0;
        res.why[(size_t)r] = h_status[i];
        res.c_off[(size_t)r] = pos + h_scan_c[i];
        res.c_len[(size_t)r] = h_scan_c[i + 1] - h_scan_c[i];
        res.l_off[(size_t)r] = pos + out_c_bytes + h_scan_l[i];
        res.l_len[(size_t)r] = h_scan_l[i + 1] - h_scan_l[i];
    }
    float ms = 0;
    cudaEventElapsedTime(&ms, w.ev[0], w.ev[1]); st.h2d += ms;
    cudaEventElapsedTime(&ms, w.ev[1], w.ev[2]); st.plan += ms;
    cudaEventElapsedTime(&ms, w.ev[2], w.ev[3]); st.kernels += ms;
    cudaEventElapsedTime(&ms, w.ev[3], w.ev[4]); st.emit += ms;
    cudaEventElapsedTime(&ms, w.ev[4], w.ev[5]); st.d2h += ms;
    return KC_OK;
}

}  // namespace

namespace {

// the candidate texts of the records in idx, record-major, as pointers into h_text and their lengths
void gather(const char *h_text, const int64_t *h_off, int32_t n, const std::vector<int64_t> &idx, std::vector<const char *> &texts,
            std::vector<int64_t> &lens) {
    texts.resize(idx.size() * n);
    lens.resize(idx.size() * n);
    for (size_t i = 0; i < idx.size(); ++i)
        for (int32_t c = 0; c < n; ++c) {
            const int64_t k = idx[i] * n + c;
            texts[i * n + c] = h_text + h_off[k];
            lens[i * n + c] = h_off[k + 1] - h_off[k];
        }
}

// The list round's alignment: the alignment pre-pass H2 (kc_align_json_batch) on host threads for the records in idx, which
// the first round marked D_LIST.  The aligned texts of the records it aligns are packed record-major into one blob from
// alloc(bytes) (off: their offsets, blob-relative; dst: their record indices); the records it declines go to `declined`.
// The element similarities of the list nodes run in one kc_alignsim pass on `device`; device < 0 runs that pass on ONE host
// thread: many times slower on a batch, faster for a few records (DESIGN.md §10).
template <class Alloc>
int align_listed(const char *h_text, const int64_t *h_off, int32_t n, int device, int32_t threads, const std::vector<int64_t> &idx, const Alloc &alloc,
                 char *&blob, std::vector<int64_t> &off, std::vector<int64_t> &dst, std::vector<int64_t> &declined) {
    const int64_t L = (int64_t)idx.size();
    std::vector<const char *> texts;
    std::vector<int64_t> lens;
    gather(h_text, h_off, n, idx, texts, lens);
    std::vector<char *> out((size_t)(L * n), nullptr);
    std::vector<int32_t> st((size_t)L, 0);
    if (const int rc = kc_align_json_batch(texts.data(), lens.data(), L, n, /*min_support_ratio=*/0.51, device, threads, out.data(), st.data(), nullptr)) {
        kc_free_strings(out.data(), L * n);  // whatever it allocated before it failed
        return rc;
    }
    off.assign(1, 0);
    dst.clear();
    declined.clear();
    for (int64_t i = 0; i < L; ++i) {
        if (st[(size_t)i] != 0) {
            declined.push_back(idx[(size_t)i]);
            continue;
        }
        dst.push_back(idx[(size_t)i]);
        for (int32_t c = 0; c < n; ++c) off.push_back(off.back() + (int64_t)strlen(out[(size_t)(i * n + c)]));
    }
    blob = alloc((size_t)off.back());
    int rc = blob ? KC_OK : kc_fail(KC_ENOMEM, "kc_consolidate_json_packed: cannot allocate %lld bytes of aligned texts", (long long)off.back());
    for (int64_t i = 0, k = 0; i < L && !rc; ++i) {
        if (st[(size_t)i] != 0) continue;
        for (int32_t c = 0; c < n; ++c, ++k) memcpy(blob + off[(size_t)k], out[(size_t)(i * n + c)], (size_t)(off[(size_t)k + 1] - off[(size_t)k]));
    }
    kc_free_strings(out.data(), L * n);
    return rc;
}

// The list round of a call (KC_JSON_LISTS): the records the first round marked D_LIST are aligned (align_listed) and the
// aligned texts consolidated by run_round with list nodes (Chunk::lists = 2) on the same workers, streams and chunking; their
// results land at the records' own indices.  What H2 declines keeps status 1 with D_ALIGN.
template <class Round>
int list_round(kc_json_result &res, const char *h_text, const int64_t *h_off, const float *h_seq, int32_t n, int device, int32_t threads,
               Round &run_round) {
    std::vector<int64_t> idx;
    for (int64_t r = 0; r < res.R; ++r)
        if (res.status[(size_t)r] && res.why[(size_t)r] == kc::js::D_LIST) idx.push_back(r);
    if (idx.empty()) return KC_OK;
    PinnedBlob texts;
    auto alloc = [&](size_t bytes) {
        texts = acquire_blob(bytes + 16);
        return texts.p;
    };
    char *blob = nullptr;
    std::vector<int64_t> off, dst, declined;
    // the similarity pass on the device pays a launch, an allocation and a synchronisation per call: a handful of records
    // (single requests) align faster with the pass on the host
    const int sim_device = idx.size() >= 64 ? device : -1;
    int rc = align_listed(h_text, h_off, n, sim_device, threads, idx, alloc, blob, off, dst, declined);
    for (int64_t r : declined) res.why[(size_t)r] = kc::js::D_ALIGN;
    const int64_t M = (int64_t)dst.size();
    if (!rc && M) {
        std::vector<float> seq;
        if (h_seq) {  // the aligned records' candidate sums, in the aligned batch's order
            seq.resize((size_t)(M * n));
            for (int64_t i = 0; i < M; ++i) memcpy(&seq[(size_t)(i * n)], h_seq + dst[(size_t)i] * n, (size_t)n * 4);
        }
        // grow the result blob to what the first round used plus the aligned round's output (no chunk is in flight between the
        // rounds).  Sized from each record's structure, not its length: a leaf's value and confidence print in at most 24
        // characters each (float.__repr__) plus their separators, so a list of small ints has likelihoods several times its text
        size_t est = 4096;  // small: a single request's aligned round fits the pooled ~1 MiB blob its first round got
        for (int64_t i = 0; i < M; ++i) {
            const char *t = blob + off[(size_t)(i * n)];
            const int64_t len = off[(size_t)(i * n + 1)] - off[(size_t)(i * n)];
            int64_t tokens = 1;  // every value ends at a ',' or a closer; every closer is a token of its own
            for (int64_t k = 0; k < len; ++k) tokens += t[k] == ',' ? 1 : (t[k] == ']' || t[k] == '}') ? 2 : 0;
            est += (size_t)(2 * len + 32 * tokens);
        }
        const size_t need = (size_t)res.used.load() + est;
        if (need > res.blob.cap) {
            PinnedBlob bigger = acquire_blob(need);
            if (!bigger.p) rc = kc_fail(KC_ENOMEM, "kc_consolidate_json_packed: cannot grow the pinned output blob to %zu bytes", need);
            else {
                memcpy(bigger.p, res.blob.p, (size_t)res.used.load());
                release_blob(res.blob);
                res.blob = bigger;
            }
        }
        if (!rc) rc = run_round(blob, off.data(), h_seq ? seq.data() : nullptr, M, (uint8_t)2, dst.data());
    }
    release_blob(texts);
    return rc;
}

}  // namespace

extern "C" {

namespace {

// kc_consolidate_json_packed, and with h_seq its likelihood-weighted variant (which hands no record to the host path: that
// path votes by count; nor does KC_JSON_NUMERIC_MEDOID: that path decides numbers the sync way)
int consolidate_packed(const char *h_text, const int64_t *h_off, const float *h_seq, int64_t n_records, int32_t n, double rel_eps,
                       double abs_eps, int device, int32_t threads, uint32_t flags, kc_json_result **out) {
    if (!out) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: NULL out");
    if (h_seq || (flags & KC_JSON_NUMERIC_MEDOID)) flags |= KC_JSON_DEVICE_ONLY;
    *out = nullptr;
    if (n < 2 || n > KC_MAX_CANDIDATES) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: n=%d outside [2,%d]", n, KC_MAX_CANDIDATES);
    if (n_records < 0 || (n_records && (!h_text || !h_off))) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: bad arguments");
    if (!(rel_eps >= 0.0) || !(abs_eps >= 0.0)) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed: rel_eps/abs_eps must be >= 0");
    const auto t_start = std::chrono::steady_clock::now();
    int prev = 0;
    KC_CUDA_I(cudaGetDevice(&prev));
    KC_CUDA_I(cudaSetDevice(device));
    int sm_count = 0, cc_major = 0;
    KC_CUDA_I(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
    KC_CUDA_I(cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, device));
    if (cc_major != 9) {
        cudaSetDevice(prev);
        return kc_fail(KC_ENODEV, "device %d has compute capability %d.x; this library is sm_90a only", device, cc_major);
    }
    kc_json_result *res = new (std::nothrow) kc_json_result;
    if (!res) return kc_fail(KC_ENOMEM, "kc_consolidate_json_packed: out of memory");
    const int64_t R = n_records;
    res->R = R;
    res->c_off.assign((size_t)R, 0);
    res->c_len.assign((size_t)R, 0);
    res->l_off.assign((size_t)R, 0);
    res->l_len.assign((size_t)R, 0);
    res->status.assign((size_t)R, 1);
    res->why.assign((size_t)R, 0);
    const int64_t total_bytes = R ? h_off[R * n] - h_off[0] : 0;
    // The consensus of a record is about one candidate long and its likelihoods about as long again (numbers can grow:
    // "5" -> "5.0", 17-digit means).  A chunk whose output does not fit what is left is handed to the host path.
    res->blob = acquire_blob((size_t)(total_bytes / n * 3 + (1 << 20)));  // small requests all ask for ~1 MiB: the pool's blobs fit
    if (!res->blob.p) {
        delete res;
        cudaSetDevice(prev);
        return kc_fail(KC_ENOMEM, "kc_consolidate_json_packed: cannot allocate the pinned output blob");
    }
    // chunks of ~chunk_mb of text; records are never split
    size_t chunk_bytes = (size_t)64 << 20;
    if (const char *e = getenv("KC_JSON_CHUNK_MB")) chunk_bytes = (size_t)std::min(1024, std::max(1, atoi(e))) << 20;  // K4's CSR offsets are int32
    int max_workers = 3;
    if (const char *e = getenv("KC_JSON_STREAMS")) max_workers = std::max(1, std::min(8, atoi(e)));
    int n_chunks = 0, n_streams = 0;
    std::vector<ChunkStage> stages((size_t)max_workers);
    // one round of chunks over a batch of Rb records (the call's, or the aligned round's), several chunks in flight
    auto run_round = [&](const char *text, const int64_t *off, const float *seq, int64_t Rb, uint8_t lists, const int64_t *dst) -> int {
        std::vector<int64_t> cuts{0};
        int64_t r = 0;
        while (r < Rb) {
            // records are a few KB: advance by estimate, then adjust
            const int64_t start = off[r * n];
            int64_t lo = r + 1, hi = Rb;
            while (lo < hi) {  // largest r1 with bytes(r, r1) <= chunk_bytes (at least one record)
                const int64_t mid = lo + (hi - lo + 1) / 2;
                if ((size_t)(off[mid * n] - start) <= chunk_bytes) lo = mid;
                else hi = mid - 1;
            }
            r = lo;
            cuts.push_back(r);
        }
        const int chunks = (int)cuts.size() - 1;
        const int n_workers = std::max(1, std::min(max_workers, chunks));
        n_chunks += chunks;
        n_streams = std::max(n_streams, n_workers);
        std::vector<Worker *> workers;
        for (int i = 0; i < n_workers; ++i) workers.push_back(acquire_worker(device));
        std::vector<int> rcs((size_t)n_workers, KC_OK);
        std::vector<std::string> errs((size_t)n_workers);
        std::atomic<int> next{0};
        auto body = [&](int wi) {
            cudaSetDevice(device);
            Worker &w = *workers[(size_t)wi];
            int rc = w.init(device);
            while (!rc) {
                const int k = next.fetch_add(1);
                if (k >= chunks) break;
                rc = run_chunk(w, text, off, seq, flags, lists, dst, cuts[(size_t)k], cuts[(size_t)k + 1], n, rel_eps, abs_eps, sm_count, *res,
                               stages[(size_t)wi]);
            }
            if (rc) {
                cudaStreamSynchronize(w.stream);
                errs[(size_t)wi] = kc_last_error();
            }
            rcs[(size_t)wi] = rc;
        };
        if (n_workers == 1) {
            body(0);
        } else {
            std::vector<std::thread> pool;
            for (int i = 0; i < n_workers; ++i) pool.emplace_back(body, i);
            for (auto &t : pool) t.join();
        }
        for (Worker *w : workers) release_worker(w);
        for (int i = 0; i < n_workers; ++i)
            if (rcs[(size_t)i]) return kc_fail(rcs[(size_t)i], "%s", errs[(size_t)i].c_str());
        return KC_OK;
    };
    const bool lists = (flags & KC_JSON_LISTS) != 0;
    int rc = run_round(h_text, h_off, h_seq, R, lists ? 1 : 0, nullptr);
    if (!rc && lists) rc = list_round(*res, h_text, h_off, h_seq, n, device, threads, run_round);
    const auto t_gpu = std::chrono::steady_clock::now();
    // the records the device path declined: host path (H1), unless the caller only wants the device path
    int64_t n_declined = 0, n_host = 0;
    if (!rc) {
        std::vector<int64_t> idx;
        for (int64_t r = 0; r < R; ++r) {
            if (!res->status[(size_t)r]) continue;
            ++n_declined;
            // what the list round's alignment declined, H1 would decline too: it runs the same pre-pass (align_values, the
            // same min_support_ratio) on the same texts before anything else
            if (res->why[(size_t)r] != kc::js::D_ALIGN) idx.push_back(r);
        }
        if (!idx.empty() && !(flags & KC_JSON_DEVICE_ONLY)) {
            const int64_t D = (int64_t)idx.size();
            std::vector<const char *> texts;
            std::vector<int64_t> lens;
            gather(h_text, h_off, n, idx, texts, lens);
            std::vector<char *> oc((size_t)D, nullptr), ol((size_t)D, nullptr);
            std::vector<uint8_t> hs((size_t)D, 1);
            rc = kc_consolidate_json(texts.data(), lens.data(), D, n, rel_eps, abs_eps, device, threads, oc.data(), ol.data(), hs.data());
            if (!rc) {
                int64_t pos = res->used.load(), extra = 0;
                for (int64_t i = 0; i < D; ++i)
                    if (hs[(size_t)i] == 0) extra += (int64_t)(strlen(oc[(size_t)i]) + strlen(ol[(size_t)i]));
                char *base = res->blob.p;
                if (pos + extra > (int64_t)res->blob.cap) {  // rare: move the texts to the heap (the pinned blob goes back to the pool)
                    res->heap.resize((size_t)(pos + extra));
                    memcpy(&res->heap[0], res->blob.p, (size_t)pos);
                    release_blob(res->blob);
                    res->blob = PinnedBlob{};
                    base = &res->heap[0];
                }
                for (int64_t i = 0; i < D; ++i) {
                    if (hs[(size_t)i] != 0) continue;
                    const int64_t r = idx[(size_t)i];
                    const size_t lc = strlen(oc[(size_t)i]), ll = strlen(ol[(size_t)i]);
                    memcpy(base + pos, oc[(size_t)i], lc);
                    memcpy(base + pos + lc, ol[(size_t)i], ll);
                    res->c_off[(size_t)r] = pos;
                    res->l_off[(size_t)r] = pos + (int64_t)lc;
                    res->c_len[(size_t)r] = (int64_t)lc;
                    res->l_len[(size_t)r] = (int64_t)ll;
                    res->status[(size_t)r] = 2;
                    pos += (int64_t)(lc + ll);
                    ++n_host;
                }
                res->used.store(pos);
            }
            kc_free_strings(oc.data(), D);
            kc_free_strings(ol.data(), D);
        }
    }
    cudaSetDevice(prev);
    if (rc) {
        release_blob(res->blob);
        delete res;
        return rc;
    }
    const auto t_end = std::chrono::steady_clock::now();
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    kc_json_stats &s = res->stats;
    s.n_records = R;
    s.n_device = R - n_declined;
    s.n_host = n_host;
    s.n_python = n_declined - n_host;
    s.input_bytes = total_bytes;
    s.output_bytes = res->used.load();
    s.chunks = n_chunks;
    s.streams = n_streams;
    for (auto &g : stages) {
        s.h2d_ms += g.h2d;
        s.plan_ms += g.plan;
        s.kernel_ms += g.kernels;
        s.emit_ms += g.emit;
        s.d2h_ms += g.d2h;
    }
    s.device_path_wall_ms = ms(t_start, t_gpu);
    s.host_path_wall_ms = ms(t_gpu, t_end);
    s.wall_ms = ms(t_start, t_end);
    *out = res;
    return KC_OK;
}

}  // namespace

int kc_consolidate_json_packed(const char *h_text, const int64_t *h_off, int64_t n_records, int32_t n, double rel_eps, double abs_eps,
                               int device, int32_t threads, uint32_t flags, kc_json_result **out) {
    return consolidate_packed(h_text, h_off, nullptr, n_records, n, rel_eps, abs_eps, device, threads, flags, out);
}

int kc_consolidate_json_packed_weighted(const char *h_text, const int64_t *h_off, const float *h_seq_logprob, int64_t n_records, int32_t n,
                                        double rel_eps, double abs_eps, int device, int32_t threads, uint32_t flags, kc_json_result **out) {
    if (n_records > 0 && !h_seq_logprob) return kc_fail(KC_EINVAL, "kc_consolidate_json_packed_weighted: NULL h_seq_logprob");
    static const float none = 0.0f;
    return consolidate_packed(h_text, h_off, h_seq_logprob ? h_seq_logprob : &none, n_records, n, rel_eps, abs_eps, device, threads, flags, out);
}

int kc_json_result_view(kc_json_result *res, const char **text, const int64_t **content_off, const int64_t **content_len,
                        const int64_t **likelihoods_off, const int64_t **likelihoods_len, const uint8_t **status, const uint8_t **why,
                        kc_json_stats *stats) {
    if (!res) return kc_fail(KC_EINVAL, "kc_json_result_view: NULL result");
    if (text) *text = res->blob.p ? res->blob.p : res->heap.data();
    if (content_off) *content_off = res->c_off.data();
    if (content_len) *content_len = res->c_len.data();
    if (likelihoods_off) *likelihoods_off = res->l_off.data();
    if (likelihoods_len) *likelihoods_len = res->l_len.data();
    if (status) *status = res->status.data();
    if (why) *why = res->why.data();
    if (stats) *stats = res->stats;
    return KC_OK;
}

void kc_json_result_free(kc_json_result *res) {
    if (!res) return;
    release_blob(res->blob);
    delete res;
}

// ---------------------------------------------------------------- test hooks: the device phases, run on the host

struct kc_debug_jsongpu {
    std::vector<int64_t> off;
    std::vector<uint8_t> text;
    int32_t n = 0;
    int64_t R = 0;
    std::vector<std::vector<uint8_t>> arrays;  // chunk_arrays (operator new aligns them for any type, Tok's 16 bytes included)
    unsigned long long counters[6] = {0, 0, 0, 0, 0, 0};
    std::vector<uint8_t> out_c, out_l;
    // KC_JSON_LISTS: records [R_out, R) are the aligned round's (record src[i - R_out] of the call); emit splices them back
    int64_t R_out = 0;
    std::vector<int64_t> src;
    std::vector<int64_t> spliced_c, spliced_l;
    std::vector<uint8_t> spliced_out_c, spliced_out_l;
    Chunk ch{};
};

int kc_debug_jsongpu_plan(const char *h_text, const int64_t *h_off, int64_t n_records, int32_t n, kc_debug_jsongpu **out) {
    return kc_debug_jsongpu_plan_flags(h_text, h_off, n_records, n, 0u, out);
}

namespace {

// the device phases of one chunk on the host, in run_chunk's order (union round included) up to A2; records [aligned0, R) in
// the aligned round
void plan_twin(kc_debug_jsongpu *h, const char *h_text, const int64_t *h_off, int64_t R, int32_t n, uint32_t flags, uint8_t lists, int32_t aligned0) {
    h->R = R;
    h->R_out = R;
    h->n = n;
    h->off.assign(h_off, h_off + R * n + 1);
    h->text.assign((const uint8_t *)h_text + h_off[0], (const uint8_t *)h_text + h_off[R * n]);
    Chunk &ch = h->ch;
    ch.text = h->text.data();
    ch.off = h->off.data();
    ch.R = (int32_t)R;
    ch.n = n;
    ch.counters = h->counters;
    set_flags(ch, flags, lists, aligned0);
    auto host = [&](int k, auto *&ptr, size_t len, size_t, int fill, bool) -> int {
        using E = std::remove_reference_t<decltype(*ptr)>;
        if (h->arrays.size() <= (size_t)k) h->arrays.resize((size_t)k + 1);
        h->arrays[(size_t)k].resize(len * sizeof(E), (uint8_t)fill);  // keeps what is there, fills the rest
        ptr = reinterpret_cast<E *>(h->arrays[(size_t)k].data());
        return KC_OK;
    };
    Units u{(size_t)R, h->text.size()};
    chunk_arrays(host, ch, RECORDS, u, 0, true);
    for (int32_t r = 0; r < R; ++r) kc::js::count_record(ch, r);
    for (int64_t r = 0; r < R; ++r) ch.slot[r + 1] = ch.slot[r] + ch.fcount[r];
    u.T = ch.slot[R];
    chunk_arrays(host, ch, SLOTS, u, 0, true);
    const kc::js::HostTeam team{team_size(n)};
    for (int32_t r = 0; r < R; ++r) kc::js::plan_step(ch, r, team);
    if ((u.P = h->counters[3])) {  // the union round, as run_chunk / union_round run it
        const int32_t P = (int32_t)u.P;
        chunk_arrays(host, ch, UNION, u, 0, true);
        ch.uslot = (uint32_t)u.T;
        for (int32_t p = 0; p < P; ++p) kc::js::union_count_step(ch, p, team);
        u.S = std::max<size_t>(h->counters[4], 1);
        chunk_arrays(host, ch, SCRATCH, u, 0, true);
        for (int32_t p = 0; p < P; ++p) kc::js::union_build_step(ch, p, team);
        const size_t keep = u.T;
        u.T += h->counters[5];
        chunk_arrays(host, ch, SLOTS, u, keep, true);
        for (int32_t p = 0; p < P; ++p) kc::js::union_plan_step(ch, p, team);
    }
    for (uint32_t *cnt : {ch.mcount, ch.scount, ch.ccount}) exclusive_scan(cnt, u.R + 1);
    chunk_arrays(host, ch, CSR, u, 0, true);
    for (int32_t r = 0; r < R; ++r) kc::js::medoid_step(ch, r, team);
}

}  // namespace

// With KC_JSON_LISTS the twin runs the list round as consolidate_packed does: the first round finds the D_LIST records, H2
// aligns them (align_listed), and the aligned texts are appended to the batch as records of the aligned round, planned in the
// same chunk behind the call's records.  The batch is planned twice on purpose: the first plan only finds the D_LIST records,
// and the second replans the call's records next to the aligned ones, so that all groups live in one set of input arrays
// (the call's records plan the same both times).  Their groups follow the first round's in every input hook; emit splices their texts
// and statuses back to the call's records.
int kc_debug_jsongpu_plan_flags(const char *h_text, const int64_t *h_off, int64_t n_records, int32_t n, uint32_t flags,
                                kc_debug_jsongpu **out) {
    if (!h_text || !h_off || !out || n < 2 || n > KC_MAX_CANDIDATES || n_records < 0) return KC_EINVAL;
    const int64_t R = n_records;
    kc_debug_jsongpu *h = new kc_debug_jsongpu;
    const bool lists = (flags & KC_JSON_LISTS) != 0;
    plan_twin(h, h_text, h_off, R, n, flags, lists ? 1 : 0, INT32_MAX);
    std::vector<int64_t> idx;
    for (int64_t r = 0; r < R && lists; ++r)
        if (h->ch.status[r] == kc::js::D_LIST) idx.push_back(r);
    if (idx.empty()) {
        *out = h;
        return KC_OK;
    }
    std::vector<char> aligned;
    auto alloc = [&](size_t bytes) {
        aligned.resize(bytes + 1);
        return aligned.data();
    };
    char *blob = nullptr;
    std::vector<int64_t> aoff, dst, declined;
    if (const int rc = align_listed(h_text, h_off, n, -1, 0, idx, alloc, blob, aoff, dst, declined)) {
        delete h;
        return rc;
    }
    const int64_t M = (int64_t)dst.size(), base = h_off[R * n] - h_off[0];
    std::vector<char> text(h_text + h_off[0], h_text + h_off[R * n]);
    text.insert(text.end(), blob, blob + aoff.back());
    std::vector<int64_t> off((size_t)((R + M) * n + 1));
    for (int64_t k = 0; k <= R * n; ++k) off[(size_t)k] = h_off[k] - h_off[0];
    for (int64_t k = 1; k <= M * n; ++k) off[(size_t)(R * n + k)] = base + aoff[(size_t)k];
    delete h;
    h = new kc_debug_jsongpu;
    plan_twin(h, text.data(), off.data(), R + M, n, flags, 1, (int32_t)R);
    h->R_out = R;
    h->src = dst;
    for (int64_t r : declined) h->ch.status[r] = kc::js::D_ALIGN;
    int32_t *vrec = h->ch.vrec;  // the aligned records' vote groups weigh with their call records' candidate sums
    for (uint64_t g = 0; g < h->counters[0]; ++g)
        if (vrec[g] >= R) vrec[g] = (int32_t)dst[(size_t)(vrec[g] - R)];
    *out = h;
    return KC_OK;
}

// the medoid groups of the planned batch in kc_medoid_str's CSR form, and where the test puts K4's results
int kc_debug_jsongpu_medoid_inputs(const kc_debug_jsongpu *h, const uint8_t **chars, const int32_t **str_off, const int32_t **grp_off,
                                   int64_t *n_groups) {
    if (!h) return KC_EINVAL;
    if (chars) *chars = h->ch.mchars;
    if (str_off) *str_off = h->ch.mstr_off;
    if (grp_off) *grp_off = h->ch.mgrp_off;
    if (n_groups) *n_groups = (int64_t)h->counters[2];
    return KC_OK;
}

int kc_debug_jsongpu_set_medoid(kc_debug_jsongpu *h, const int32_t *medoid_idx, const double *medoid_avg) {
    if (!h) return KC_EINVAL;
    h->ch.midx = medoid_idx;  // must stay alive until kc_debug_jsongpu_emit has returned
    h->ch.mavg = medoid_avg;
    return KC_OK;
}

int kc_debug_jsongpu_set_numeric_medoid(kc_debug_jsongpu *h, const int32_t *best, const double *best_avg) {
    if (!h) return KC_EINVAL;
    h->ch.xbest = best;  // must stay alive until kc_debug_jsongpu_emit has returned
    h->ch.xavg = best_avg;
    return KC_OK;
}

int kc_debug_jsongpu_inputs(const kc_debug_jsongpu *h, const int8_t **vote_cells, int64_t *n_vote_groups, const double **num_cells,
                            int64_t *n_num_groups, const uint8_t **status) {
    if (!h) return KC_EINVAL;
    if (vote_cells) *vote_cells = h->ch.vcells;
    if (n_vote_groups) *n_vote_groups = (int64_t)h->counters[0];
    if (num_cells) *num_cells = h->ch.xcells;
    if (n_num_groups) *n_num_groups = (int64_t)h->counters[1];
    if (status) *status = h->ch.status;
    return KC_OK;
}

int kc_debug_jsongpu_emit(kc_debug_jsongpu *h, const uint32_t *vote_meta, const double *num_value, const uint32_t *num_meta,
                          const char **content, const int64_t **content_off, const char **likelihoods, const int64_t **likelihoods_off) {
    return kc_debug_jsongpu_emit_weighted(h, vote_meta, nullptr, num_value, num_meta, content, content_off, likelihoods, likelihoods_off);
}

int kc_debug_jsongpu_group_records(const kc_debug_jsongpu *h, const int32_t **group_record) {
    if (!h) return KC_EINVAL;
    if (group_record) *group_record = h->ch.vrec;
    return KC_OK;
}

int kc_debug_jsongpu_emit_weighted(kc_debug_jsongpu *h, const uint32_t *vote_meta, const float *vote_weight, const double *num_value,
                                   const uint32_t *num_meta, const char **content, const int64_t **content_off, const char **likelihoods,
                                   const int64_t **likelihoods_off) {
    if (!h) return KC_EINVAL;
    Chunk &ch = h->ch;
    ch.vmeta = vote_meta;
    ch.vweight = vote_weight;
    ch.xvalue = num_value;
    ch.xmeta = num_meta;
    const int64_t R = h->R;
    const kc::js::HostTeam team{team_size(h->n)};
    for (int32_t r = 0; r < R; ++r) kc::js::len_step(ch, r, team);
    exclusive_scan(ch.len_c, (size_t)R + 1);
    exclusive_scan(ch.len_l, (size_t)R + 1);
    const int64_t ac = ch.len_c[R], al = ch.len_l[R];
    h->out_c.assign((size_t)std::max<int64_t>(ac, 1), 0);
    h->out_l.assign((size_t)std::max<int64_t>(al, 1), 0);
    ch.out_c = h->out_c.data();
    ch.out_l = h->out_l.data();
    for (int32_t r = 0; r < R; ++r) kc::js::write_step(ch, r, team);
    if (h->R_out < R) {  // the list round: each aligned record's texts and status go to its call record
        const int64_t Ro = h->R_out;
        std::vector<int64_t> from((size_t)Ro);
        for (int64_t r = 0; r < Ro; ++r) from[(size_t)r] = r;
        for (int64_t i = 0; i < R - Ro; ++i) {
            from[(size_t)h->src[(size_t)i]] = Ro + i;
            ch.status[h->src[(size_t)i]] = ch.status[Ro + i];
        }
        auto splice = [&](const int64_t *o, const std::vector<uint8_t> &blob, std::vector<int64_t> &so, std::vector<uint8_t> &sb) {
            so.assign((size_t)Ro + 1, 0);
            sb.clear();
            for (int64_t r = 0; r < Ro; ++r) {
                const int64_t k = from[(size_t)r];
                sb.insert(sb.end(), blob.begin() + o[(size_t)k], blob.begin() + o[(size_t)k + 1]);
                so[(size_t)r + 1] = (int64_t)sb.size();
            }
            sb.push_back(0);
        };
        splice(ch.len_c, h->out_c, h->spliced_c, h->spliced_out_c);
        splice(ch.len_l, h->out_l, h->spliced_l, h->spliced_out_l);
        if (content) *content = (const char *)h->spliced_out_c.data();
        if (content_off) *content_off = h->spliced_c.data();
        if (likelihoods) *likelihoods = (const char *)h->spliced_out_l.data();
        if (likelihoods_off) *likelihoods_off = h->spliced_l.data();
        return KC_OK;
    }
    if (content) *content = (const char *)h->out_c.data();
    if (content_off) *content_off = ch.len_c;
    if (likelihoods) *likelihoods = (const char *)h->out_l.data();
    if (likelihoods_off) *likelihoods_off = ch.len_l;
    return KC_OK;
}

void kc_debug_jsongpu_free(kc_debug_jsongpu *h) { delete h; }

// float(text) and float.__repr__ as the device code computes them (batch test hooks)
int kc_debug_parse_doubles(const char *text, const int64_t *off, int64_t count, double *out, uint8_t *ok) {
    if (!text || !off || !out || !ok) return KC_EINVAL;
    for (int64_t i = 0; i < count; ++i) {
        double v = 0.0;
        ok[i] = kc::js::to_double((const uint8_t *)text + off[i], (uint32_t)(off[i + 1] - off[i]), v) ? 1 : 0;
        out[i] = v;
    }
    return KC_OK;
}

int kc_debug_float_reprs(const double *xs, int64_t count, char *out /* [count][32] */, int32_t *lens) {
    if (!xs || !out || !lens) return KC_EINVAL;
    for (int64_t i = 0; i < count; ++i) {
        kc::js::Sink s{(uint8_t *)out + i * 32, 0};
        kc::js::float_repr(xs[i], s);
        lens[i] = (int32_t)s.n;
    }
    return KC_OK;
}

int kc_debug_round5(const double *xs, int64_t count, double *out) {
    if (!xs || !out) return KC_EINVAL;
    for (int64_t i = 0; i < count; ++i) out[i] = kc::py_round5(xs[i]);
    return KC_OK;
}

}  // extern "C"

// ---------------------------------------------------------------- the number conversions' device instantiation (test hooks)

namespace {

__global__ void parse_doubles_kernel(const uint8_t *__restrict__ text, const int64_t *__restrict__ off, int64_t count, double *__restrict__ out,
                                     uint8_t *__restrict__ ok) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        double v = 0.0;
        ok[i] = kc::js::to_double(text + off[i], (uint32_t)(off[i + 1] - off[i]), v) ? 1 : 0;
        out[i] = v;
    }
}

__global__ void float_reprs_kernel(const double *__restrict__ xs, int64_t count, uint8_t *__restrict__ out, int32_t *__restrict__ lens) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        kc::js::Sink s{out + i * 32, 0};
        kc::js::float_repr(xs[i], s);
        lens[i] = (int32_t)s.n;
    }
}

constexpr int kDebugBlock = 256, kDebugGrid = 264;  // a grid stride of 67,584 threads: large batches loop

}  // namespace

extern "C" {

// kc_debug_parse_doubles / kc_debug_float_reprs with the conversions run on `device`, one thread per value
int kc_debug_parse_doubles_device(const char *text, const int64_t *off, int64_t count, double *out, uint8_t *ok, int device) {
    if (!text || !off || !out || !ok || count < 0) return KC_EINVAL;
    if (count == 0) return KC_OK;
    KC_CUDA_I(cudaSetDevice(device));
    const size_t n_text = (size_t)off[count];
    kc::Staged st("kc_debug_parse_doubles_device");
    uint8_t *d[4];  // text, offsets, values, flags
    R_(st.alloc({n_text, ((size_t)count + 1) * 8, (size_t)count * 8, (size_t)count}, d));
    if (n_text) KC_CUDA_I(cudaMemcpyAsync(d[0], text, n_text, cudaMemcpyHostToDevice, st.stream));
    KC_CUDA_I(cudaMemcpyAsync(d[1], off, ((size_t)count + 1) * 8, cudaMemcpyHostToDevice, st.stream));
    parse_doubles_kernel<<<kDebugGrid, kDebugBlock, 0, st.stream>>>(d[0], reinterpret_cast<const int64_t *>(d[1]), count,
                                                                   reinterpret_cast<double *>(d[2]), d[3]);
    KC_CUDA_I(cudaGetLastError());
    KC_CUDA_I(cudaMemcpyAsync(out, d[2], (size_t)count * 8, cudaMemcpyDeviceToHost, st.stream));
    KC_CUDA_I(cudaMemcpyAsync(ok, d[3], (size_t)count, cudaMemcpyDeviceToHost, st.stream));
    return st.finish();
}

int kc_debug_float_reprs_device(const double *xs, int64_t count, char *out /* [count][32] */, int32_t *lens, int device) {
    if (!xs || !out || !lens || count < 0) return KC_EINVAL;
    if (count == 0) return KC_OK;
    KC_CUDA_I(cudaSetDevice(device));
    kc::Staged st("kc_debug_float_reprs_device");
    uint8_t *d[3];  // values, texts, lengths
    R_(st.alloc({(size_t)count * 8, (size_t)count * 32, (size_t)count * 4}, d));
    KC_CUDA_I(cudaMemcpyAsync(d[0], xs, (size_t)count * 8, cudaMemcpyHostToDevice, st.stream));
    float_reprs_kernel<<<kDebugGrid, kDebugBlock, 0, st.stream>>>(reinterpret_cast<const double *>(d[0]), count, d[1],
                                                                 reinterpret_cast<int32_t *>(d[2]));
    KC_CUDA_I(cudaGetLastError());
    KC_CUDA_I(cudaMemcpyAsync(out, d[1], (size_t)count * 32, cudaMemcpyDeviceToHost, st.stream));
    KC_CUDA_I(cudaMemcpyAsync(lens, d[2], (size_t)count * 4, cudaMemcpyDeviceToHost, st.stream));
    return st.finish();
}

}  // extern "C"

// ---------------------------------------------------------------- bench / test input: schema S32 as candidate texts

namespace {

struct SplitMix {
    uint64_t s;
    uint64_t next() {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    double uni() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

// One record of schema S32 (SURVEY.md §8d; same distribution as k_llms_b200/synth.py): n candidate texts exactly as
// json.dumps(dict) prints them.  f00-f15 string-enum (8 words, 4 spellings that sanitise alike), f16-f23 bool, f24-f29 int in
// [1, 1e6), f30-f31 float U(1, 1e4); per field a truth, each candidate copies it w.p. p_agree, then is None w.p. p_none.
void s32_record(uint64_t seed, int64_t r, int32_t n, kc::js::Sink &o, int64_t *off /* n+1 entries, relative to o.n at entry */) {
    static const char *vocab[8] = {"alpha", "Bravo", "charlie", "DELTA", "echo", "foxtrot", "golf", "Hotel"};
    SplitMix g{seed * 0x9E3779B97F4A7C15ull + (uint64_t)r * 0xD1B54A32D192ED03ull + 1};
    const double p_agree = 0.8, p_none = 0.05;
    int32_t truth_code[24];
    double truth_num[8];
    for (int f = 0; f < 24; ++f) truth_code[f] = (int32_t)(g.uni() * (f < 16 ? 8 : 2));
    for (int f = 0; f < 8; ++f) truth_num[f] = f < 6 ? (double)(int64_t)(1 + g.uni() * (1e6 - 1)) : 1.0 + g.uni() * (1e4 - 1.0);
    const int64_t base = o.n;
    for (int32_t c = 0; c < n; ++c) {
        off[c] = o.n - base;
        o.put('{');
        for (int f = 0; f < 32; ++f) {
            if (f) o.lit(", ");
            o.lit("\"f");
            o.put((uint8_t)('0' + f / 10));
            o.put((uint8_t)('0' + f % 10));
            o.lit("\": ");
            const bool agree = g.uni() < p_agree, none = g.uni() < p_none;
            if (f < 24) {
                const int32_t draw = (int32_t)(g.uni() * (f < 16 ? 8 : 2));
                const int32_t k = agree ? truth_code[f] : draw;
                if (none) {
                    o.lit("null");
                } else if (f >= 16) {
                    o.lit(k ? "true" : "false");
                } else {
                    const char *w = vocab[k];
                    const int variant = (int)((r + c + f) & 3);
                    o.put('"');
                    if (variant == 3) o.put(' ');
                    for (const char *q = w; *q; ++q) {
                        char ch = *q;
                        if (variant == 1 && ch >= 'a' && ch <= 'z') ch = (char)(ch - 32);
                        if (variant == 2 && ch >= 'A' && ch <= 'Z') ch = (char)(ch + 32);
                        o.put((uint8_t)ch);
                    }
                    if (variant == 2) o.put('!');
                    o.put('"');
                }
            } else {
                const int k = f - 24;
                const double draw = k < 6 ? (double)(int64_t)(1 + g.uni() * (1e6 - 1)) : 1.0 + g.uni() * (1e4 - 1.0);
                const double v = agree ? truth_num[k] : draw;
                if (none) {
                    o.lit("null");
                } else if (k < 6) {
                    char buf[24];
                    const int len = snprintf(buf, sizeof buf, "%lld", (long long)v);
                    o.put((const uint8_t *)buf, (uint32_t)len);
                } else {
                    kc::js::float_repr(v, o);
                }
            }
        }
        o.put('}');
    }
    off[n] = o.n - base;
}

}  // namespace

extern "C" int kc_debug_s32_texts(uint64_t seed, int64_t n_records, int32_t n, int32_t threads, char *out, int64_t cap, int64_t *off) {
    if (n_records < 0 || n < 1 || n > KC_MAX_CANDIDATES || !off) return KC_EINVAL;
    if (threads <= 0) threads = (int)std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
    const int64_t R = n_records;
    const bool write = out != nullptr;
    // pass 1 (out == NULL): lengths -> off[] (absolute, off[0] = 0); pass 2: the texts, at the offsets pass 1 left in off[]
    std::atomic<int64_t> next{0};
    std::atomic<int> bad{0};
    auto body = [&] {
        std::vector<int64_t> rel((size_t)n + 1);
        for (;;) {
            const int64_t b = next.fetch_add(1024);
            if (b >= R) return;
            const int64_t e = std::min(R, b + 1024);
            for (int64_t r = b; r < e; ++r) {
                if (!write) {
                    kc::js::Sink s{nullptr, 0};
                    s32_record(seed, r, n, s, rel.data());
                    for (int32_t c = 0; c < n; ++c) off[r * n + c + 1] = rel[(size_t)c + 1] - rel[(size_t)c];  // lengths for now
                } else {
                    if (off[(r + 1) * n] > cap) {
                        bad = 1;
                        return;
                    }
                    kc::js::Sink s{(uint8_t *)out + off[r * n], 0};
                    s32_record(seed, r, n, s, rel.data());
                }
            }
        }
    };
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) pool.emplace_back(body);
    for (auto &t : pool) t.join();
    if (!write) {
        off[0] = 0;
        for (int64_t i = 1; i <= R * n; ++i) off[i] += off[i - 1];
    }
    return bad ? KC_EINVAL : KC_OK;
}
