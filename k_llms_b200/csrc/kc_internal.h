// kc_internal.h — helpers shared by the translation units of libkllms_b200.so (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

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
// diagonal).  device >= 0: one kernel launch on that device; device < 0: the same phase instantiated on the host.
// *pairs (optional) = element pairs a < b the phase decided.
extern "C" __attribute__((visibility("hidden"))) int kc_alignsim(const KcAsNode *nodes, int64_t n_nodes, const KcAsVal *vals, int64_t n_vals,
                                                                 const uint8_t *chars, int64_t n_chars, double *h_out, int64_t n_out,
                                                                 int device, int64_t *pairs);

#define KC_CUDA_I(call)                                                                                               \
    do {                                                                                                              \
        cudaError_t e_ = (call);                                                                                      \
        if (e_ != cudaSuccess) return kc_fail(KC_ECUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)
