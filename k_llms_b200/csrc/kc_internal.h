// kc_internal.h — helpers shared by the translation units of libkllms_b200.so (not part of the C ABI), among them the one
// owner of the library's device and page-locked host allocations (at the end).
//
// It also holds the one copy of each small CPython rule that the kernels and the host code must apply bit for bit
// (kc_json.cpp is host C++ and cannot include the .cuh headers, so these live here, __host__ __device__):
//     py_round5            round(x, 5)                                 (consensus_utils.py:982,1178,1187,1219)
//     confidence           the confidence of a vote / numeric result word (cu:971-982,1085-1086,1116,1177-1219,1396,1402)
//     medoid_confidence    the confidence of a similarity medoid        (cu:1085-1086,1233-1237)
//     weighted_vote_confidence  the likelihood of a likelihood-weighted vote leaf (self-defined, DESIGN.md §5)
//     py_isclose           math.isclose(a, b, rel_tol=0.01)             (cu:827-841)
//     kSimFloor            SIMILARITY_SCORE_LOWER_BOUND                 (cu:78)
// float.__repr__ is kc::js::float_repr (kc_jsoncore.cuh); the edit distance is kc_levenshtein (kc_json.cpp) on the host
// and K4's Myers loop (kc_medoid.cuh) on the device.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <initializer_list>
#include <utility>

#include "../../include/kllms_b200.h"

#ifdef __CUDACC__
#define KC_HD __host__ __device__
#else
#define KC_HD
#endif

namespace kc {

KC_HD inline uint64_t umul64hi(uint64_t a, uint64_t b) {  // the high 64 bits of a * b
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// CPython float.__round__(x, 5) (Objects/floatobject.c double_round: dtoa mode 3, i.e. the EXACT binary value rounded
// half-even to 5 decimals, then strtod).  x = mant * 2^-sh exactly; q = x * 1e5 rounded half-even in integer arithmetic on
// two 64-bit halves; q / 1e5 in IEEE double is the double nearest to the decimal q * 10^-5, which is what strtod returns.
// Domain: finite x >= 0 and below 2^46 (every confidence is in [0, 1]).  Zero, NaN and infinities come back unchanged.
KC_HD inline double py_round5(double x) {
    uint64_t bits;
    memcpy(&bits, &x, 8);
    const int biased = (int)((bits >> 52) & 0x7FF);
    uint64_t mant = bits & 0xFFFFFFFFFFFFFull;
    int exp2;  // x = mant * 2^exp2
    if (biased == 0) {
        exp2 = -1074;
    } else {
        mant |= 1ull << 52;
        exp2 = biased - 1075;
    }
    if (mant == 0) return x;
    if (exp2 >= 0) return x;  // integer-valued: nothing to round
    const int sh = -exp2;     // >= 1
    if (sh >= 128) return 0.0;
    const uint64_t lo = mant * 100000ull;  // low 64 bits of the 70-bit product
    const uint64_t hi = umul64hi(mant, 100000ull);
    uint64_t q, rem_hi, rem_lo, half_hi, half_lo;
    if (sh >= 64) {
        const int s = sh - 64;  // 0..63
        q = s == 0 ? hi : (hi >> s);
        rem_hi = s == 0 ? 0 : (hi & ((1ull << s) - 1));
        rem_lo = lo;
        half_hi = s == 0 ? 0 : (1ull << (s - 1));
        half_lo = s == 0 ? (1ull << 63) : 0;
    } else {
        q = (hi << (64 - sh)) | (lo >> sh);  // sh in 1..63; hi < 2^6 so no bits are lost for sh >= 6,
                                             // and for sh < 6 the product fits 64 bits only if hi == 0 (x >= 2^46: outside the domain)
        rem_hi = 0;
        rem_lo = lo & ((1ull << sh) - 1);
        half_hi = 0;
        half_lo = 1ull << (sh - 1);
    }
    const bool gt = rem_hi > half_hi || (rem_hi == half_hi && rem_lo > half_lo);
    const bool eq = rem_hi == half_hi && rem_lo == half_lo;
    if (gt || (eq && (q & 1))) ++q;
    return (double)q / 100000.0;
}

// The confidence the reference attaches to the consensus value of a vote (numeric == false) or numeric group, from its
// result word (KC_META_*) and the parent's valid fraction pvf.  Every operation is one IEEE operation in this order.
KC_HD inline double confidence(uint32_t m, bool numeric, double pvf) {
    const double support = (double)KC_META_SUPPORT(m), nn = (double)KC_META_NN(m), present = (double)KC_META_PRESENT(m);
    const uint32_t flags = KC_META_FLAGS(m);
    if (flags & KC_FLAG_HAS_VALUE) {
        if (!numeric) return py_round5(pvf * (support / present));  // cu:973,982
        if (flags & KC_FLAG_SINGLE) return pvf * (1.0 / present) * 1.0;  // cu:1444,1086 (unrounded)
        return py_round5(support / nn);  // cu:1177-1178,1186-1187,1218-1219
    }
    if (flags & KC_FLAG_NO_FINITE) return pvf * (nn / present);  // cu:1444,1116
    return present == 0.0 ? pvf : 0.0;  // cu:1396 / cu:1402
}

// The likelihood of a likelihood-weighted vote leaf (DESIGN.md §5, self-defined): pvf times K3b's fp32 weight (the winning
// class's share of the voting weight), rounded like every vote confidence.  The Python epilogue (columnar.Plan.materialise)
// computes the same round(pvf * float(w), 5).
KC_HD inline double weighted_vote_confidence(double pvf, float weight) { return py_round5(pvf * (double)weight); }

// The confidence of a similarity medoid among the `live` non-None strings of n candidates, avg = the medoid's mean
// similarity: cu:1444 then cu:1085-1086 (one string: itself, unrounded) or cu:1233-1237 (the medoid, rounded).
KC_HD inline double medoid_confidence(uint32_t live, int32_t n, double avg) {
    const double sub = 1.0 * ((double)live / (double)n);
    return live >= 2 ? py_round5(sub * avg) : sub * (1.0 / 1.0);
}

constexpr double kSimFloor = 1e-8;  // SIMILARITY_SCORE_LOWER_BOUND, cu:78

KC_HD inline bool py_isclose(double a, double b) {  // math.isclose(a, b, rel_tol=0.01), numerical_similarity cu:827-841
    if (a == b) return true;
    if (fabs(a) == INFINITY || fabs(b) == INFINITY) return false;
    const double diff = fabs(b - a);
    return diff <= fabs(0.01 * b) || diff <= fabs(0.01 * a);
}

}  // namespace kc

// records the thread-local text kc_last_error() returns and hands `code` back
__attribute__((visibility("hidden"))) int kc_fail(int code, const char *fmt, ...) __attribute__((format(printf, 2, 3)));

// ---- the value table of the alignment similarity phase (kc_alignsim.cuh), filled by the H2 host code (kc_json.cpp)
enum KcAsType : uint8_t { KC_AS_NONE = 0, KC_AS_BOOL, KC_AS_INT, KC_AS_FLOAT, KC_AS_STR, KC_AS_DICT, KC_AS_OTHER };
enum : uint8_t { KC_AS_FALSY = 1, KC_AS_BIGINT = 2 };

// One list element, or one member value of a flat dict element.
struct KcAsVal {
    double num;        // bool (0 / 1), int (float(v)), float
    int64_t ikey;      // int: its value when the decimal text fits in int64 (else KC_AS_BIGINT is set)
    int32_t off, len;  // str: normalised text chars[off, off + len); dict: member values [off, off + len) in key order
    int32_t raw_len;   // str: length of the raw text
    int32_t raw_id;    // str: equal raw texts <=> equal ids (within a node)
    int32_t key;       // dict member: rank of its key in the sorted keys of the node
    uint8_t type;      // KcAsType; KC_AS_OTHER: lists and dicts holding dicts or lists (not modelled)
    uint8_t flags;     // KC_AS_FALSY (`not bool(v)`), KC_AS_BIGINT
};

// One list node: T elements vals[val0 .. val0 + T) (the candidates' lists back to back) -> its dense T x T matrix at out.
struct KcAsNode {
    int64_t val0, out;
    int32_t T;
};

// Similarity matrices of the nodes into h_out (host memory; NaN where the phase does not model the pair, and on the
// diagonal).  device >= 0: one kernel launch on that device; device < 0: the same phase instantiated on the host, each node's
// pairs split over `host_lanes` lanes run one after another (1 in the product; 32 walks the pairs as a warp does).
// *pairs (optional) = element pairs a < b the phase decided.
extern "C" __attribute__((visibility("hidden"))) int kc_alignsim(const KcAsNode *nodes, int64_t n_nodes, const KcAsVal *vals, int64_t n_vals,
                                                                 const uint8_t *chars, int64_t n_chars, double *h_out, int64_t n_out,
                                                                 int device, int host_lanes, int64_t *pairs);

#define KC_CUDA_I(call)                                                                                               \
    do {                                                                                                              \
        cudaError_t e_ = (call);                                                                                      \
        if (e_ != cudaSuccess) return kc_fail(KC_ECUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// ---- device and page-locked host memory of the library (host code only).  Every cudaMalloc, cudaFree, cudaHostAlloc and
// cudaFreeHost of libkllms_b200.so is in the four functions below; a failed allocation clears CUDA's last error and reports
// KC_ENOMEM.  Owners of these allocations that live in pools are never destroyed: no CUDA call may run from a static
// destructor, after the CUDA runtime may have been torn down.
namespace kc {

inline int device_alloc(void **p, size_t bytes, const char *who) {
    if (cudaMalloc(p, bytes) == cudaSuccess) return KC_OK;
    cudaGetLastError();
    *p = nullptr;
    return kc_fail(KC_ENOMEM, "%s: cudaMalloc(%zu) failed", who, bytes);
}
inline void device_free(void *p) {
    if (p) cudaFree(p);
}
inline int pinned_alloc(void **p, size_t bytes, const char *who) {
    if (cudaHostAlloc(p, bytes, cudaHostAllocDefault) == cudaSuccess) return KC_OK;
    cudaGetLastError();
    *p = nullptr;
    return kc_fail(KC_ENOMEM, "%s: cudaHostAlloc(%zu) failed", who, bytes);
}
inline void pinned_free(void *p) {
    if (p) cudaFreeHost(p);
}

enum class Mem { Device, Pinned };

// A grow-only buffer of device or page-locked host memory.  It reallocates only when a request exceeds its capacity, and
// then with an eighth more plus 256 bytes, so that sizes that creep up from call to call do not reallocate every call.
template <Mem M>
struct GrowBuf {
    void *p = nullptr;
    size_t cap = 0;
    GrowBuf() = default;
    GrowBuf(GrowBuf &&o) noexcept : p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    ~GrowBuf() { release(); }
    void release() {
        M == Mem::Device ? device_free(p) : pinned_free(p);
        p = nullptr;
        cap = 0;
    }
    // at least `need` bytes; the contents are not kept
    int reserve(size_t need) {
        if (p && need <= cap) return KC_OK;
        release();
        const size_t bytes = need + need / 8 + 256;
        if (const int rc = M == Mem::Device ? device_alloc(&p, bytes, "device buffer") : pinned_alloc(&p, bytes, "pinned buffer")) return rc;
        cap = bytes;
        return KC_OK;
    }
    // reserve() that keeps the first `keep` bytes (device memory only): they are copied on stream s, and s is synchronised
    // before the old allocation is freed.  The old allocation is freed on every path.
    int grow(size_t need, size_t keep, cudaStream_t s) {
        static_assert(M == Mem::Device, "grow() copies device memory");
        if (!keep || (p && need <= cap)) return reserve(need);
        GrowBuf old = std::move(*this);
        if (const int rc = reserve(need)) return rc;
        if (old.p) KC_CUDA_I(cudaMemcpyAsync(p, old.p, keep < old.cap ? keep : old.cap, cudaMemcpyDeviceToDevice, s));
        KC_CUDA_I(cudaStreamSynchronize(s));
        return KC_OK;
    }
    template <typename T>
    T *as() const { return static_cast<T *>(p); }
};

// One synchronous call that uploads its inputs, launches and downloads its results: one device allocation cut into parts
// that each start 256-byte aligned, one non-blocking stream, and the call's first error in rc (where the caller also stores
// the code of a launcher it calls).  finish() waits for the stream and returns rc; the destructor destroys the stream and
// frees the allocation.
struct Staged {
    const char *who;
    void *base = nullptr;
    cudaStream_t stream = nullptr;
    int rc = KC_OK;
    explicit Staged(const char *who_) : who(who_) {}
    Staged(const Staged &) = delete;
    void operator=(const Staged &) = delete;
    ~Staged() {
        if (stream) cudaStreamDestroy(stream);
        device_free(base);
    }
    // parts[i] = the part of sizes[i] bytes; then the stream
    int alloc(std::initializer_list<size_t> sizes, uint8_t **parts) {
        auto up = [](size_t b) { return (b + 255) & ~size_t(255); };
        size_t end = 0;
        for (size_t b : sizes) end = up(end) + b;
        if (const int e = device_alloc(&base, end, who)) return e;
        end = 0;
        for (size_t b : sizes) {
            *parts++ = static_cast<uint8_t *>(base) + up(end);
            end = up(end) + b;
        }
        check(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking), "stream");
        return rc;
    }
    void check(cudaError_t e, const char *what) {
        if (e != cudaSuccess && rc == KC_OK) rc = kc_fail(KC_ECUDA, "%s: %s: %s", who, what, cudaGetErrorString(e));
    }
    int finish() {
        check(cudaStreamSynchronize(stream), "sync");
        return rc;
    }
};

}  // namespace kc
