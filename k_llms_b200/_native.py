"""ctypes binding of libkllms_b200.so — the C ABI declared in include/kllms_b200.h.

This is the ONLY compute path of the package: there is no CPU fallback.  If the shared library has not
been built (`python -c "import __graft_entry__ as g; g.build()"` or `make -C k_llms_b200/csrc`) or no
sm_90 (H100) device is visible, the functions below raise — loudly — instead of computing on the host.

torch is used for device memory and streams only (plumbing); the ABI itself takes raw pointers.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KLLMS_B200_LIB") or os.path.join(_HERE, "libkllms_b200.so")

KC_OK, KC_EINVAL, KC_ECUDA, KC_ENODEV, KC_ENOMEM = 0, -1, -2, -3, -4
MAX_CANDIDATES = 64
CODE_NONE, CODE_ABSENT = -1, -2
F64_NONE_BITS = 0x7FF8C0DE00000000
F64_ABSENT_BITS = 0x7FF8C0DF00000000
FLAG_HAS_VALUE, FLAG_SINGLE, FLAG_TIE, FLAG_NO_FINITE = 1, 2, 4, 8
OUT_LOCAL, OUT_MULTIMEM, OUT_PEERS = 0, 1, 2

_vp, _i32, _i64, _u32, _u64, _f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_double
_int, _str, _pp = ctypes.c_int, ctypes.c_char_p, ctypes.POINTER(ctypes.c_void_p)
_CONSENSUS_HOST = [_vp, _i32, _vp, _vp, _i32, _i64, _i32, _f64, _f64, _vp, _vp, _vp, _vp, _int, _vp]

# Every function of the C ABI (include/kllms_b200.h): name -> (restype, argtypes).  None is void.
_SIGNATURES = {
    "kc_version": (_int, []),
    "kc_last_error": (_str, []),
    "kc_device_count": (_int, []),
    "kc_sm_count": (_int, [_int]),
    "kc_set_device": (_int, [_int]),
    "kc_vote_i32": (_int, [_vp, _i64, _i32, _vp, _i32, _vp, _vp, _vp]),
    "kc_vote_i32_ex": (_int, [_vp, _i64, _i32, _vp, _i32, _vp, _vp, _u32, _vp]),
    "kc_vote_i32_peers": (_int, [_vp, _i64, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _vp]),
    "kc_vote_i32_peers_packed": (_int, [_vp, _i64, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "kc_vote_i32_wire": (_int, [_vp, _i64, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "kc_vote_i8": (_int, [_vp, _i64, _i32, _vp, _i32, _vp, _vp, _vp]),
    "kc_numeric_f64": (_int, [_vp, _i64, _i32, _f64, _f64, _vp, _vp, _vp]),
    "kc_numeric_f64_ex": (_int, [_vp, _i64, _i32, _f64, _f64, _vp, _vp, _u32, _vp]),
    "kc_numeric_f64_peers": (_int, [_vp, _i64, _i32, _f64, _f64, _vp, _vp, _i32, _vp, _vp]),
    "kc_push_results": (_int, [_vp, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp]),
    "kc_confidence_f64": (_int, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "kc_logprob_sum_f32": (_int, [_vp, _vp, _i64, _vp, _vp]),
    "kc_weighted_vote_i32": (_int, [_vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "kc_weighted_vote_groups_i8": (_int, [_vp, _i64, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "kc_consensus_host": (_int, _CONSENSUS_HOST),
    "kc_consensus_host_i8": (_int, _CONSENSUS_HOST),
    "kc_host_alloc": (_vp, [_u64]),
    "kc_host_free": (None, [_vp]),
    "kc_medoid_str": (_int, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "kc_medoid_str_method": (_int, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp]),
    "kc_medoid_str_host": (_int, [_vp, _i64, _vp, _vp, _i64, _i32, _vp, _vp, _int]),
    "kc_numeric_medoid_f64": (_int, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "kc_levenshtein": (_int, [_str, _i32, _str, _i32]),
    "kc_consolidate_json": (_int, [_vp, _vp, _i64, _i32, _f64, _f64, _int, _i32, _vp, _vp, _vp]),
    "kc_free_strings": (None, [_vp, _i64]),
    "kc_align_json": (_int, [ctypes.POINTER(_str), _vp, _i32, _f64, ctypes.POINTER(_str)]),
    "kc_align_json_batch": (_int, [_vp, _vp, _i64, _i32, _f64, _int, _i32, _vp, _vp, _vp]),
    "kc_json_plan": (_int, [_vp, _vp, _i64, _i32, _i32, _pp]),
    "kc_json_inputs": (_int, [_vp] * 10),
    "kc_json_emit": (_int, [_vp] * 9),
    "kc_json_free": (None, [_vp]),
    "kc_consolidate_json_packed": (_int, [_vp, _vp, _i64, _i32, _f64, _f64, _int, _i32, _u32, _pp]),
    "kc_consolidate_json_packed_weighted": (_int, [_vp, _vp, _vp, _i64, _i32, _f64, _f64, _int, _i32, _u32, _pp]),
    "kc_json_result_view": (_int, [_vp] + [_pp] * 7 + [_vp]),
    "kc_json_result_free": (None, [_vp]),
    "kc_debug_similarity_json": (_int, [_str, _str, ctypes.POINTER(_f64)]),
    "kc_debug_lsap": (_int, [_i32, _i32, _vp, _vp, _vp]),
    "kc_debug_alignsim": (_int, [_vp, _i32, _vp]),
    "kc_debug_alignsim_nodes": (_int, [_vp, _vp, _i32, _i32, _int, _vp]),
    "kc_debug_jsongpu_plan": (_int, [_vp, _vp, _i64, _i32, _pp]),
    "kc_debug_jsongpu_plan_flags": (_int, [_vp, _vp, _i64, _i32, _u32, _pp]),
    "kc_debug_jsongpu_inputs": (_int, [_vp] * 6),
    "kc_debug_jsongpu_emit": (_int, [_vp, _vp, _vp, _vp] + [_pp] * 4),
    "kc_debug_jsongpu_group_records": (_int, [_vp, _pp]),
    "kc_debug_jsongpu_emit_weighted": (_int, [_vp, _vp, _vp, _vp, _vp] + [_pp] * 4),
    "kc_debug_jsongpu_medoid_inputs": (_int, [_vp] + [_pp] * 3 + [ctypes.POINTER(_i64)]),
    "kc_debug_jsongpu_set_medoid": (_int, [_vp, _vp, _vp]),
    "kc_debug_jsongpu_set_numeric_medoid": (_int, [_vp, _vp, _vp]),
    "kc_debug_jsongpu_free": (None, [_vp]),
    "kc_debug_parse_doubles": (_int, [_vp, _vp, _i64, _vp, _vp]),
    "kc_debug_float_reprs": (_int, [_vp, _i64, _vp, _vp]),
    "kc_debug_parse_doubles_device": (_int, [_vp, _vp, _i64, _vp, _vp, _int]),
    "kc_debug_float_reprs_device": (_int, [_vp, _i64, _vp, _vp, _int]),
    "kc_debug_round5": (_int, [_vp, _i64, _vp]),
    "kc_debug_s32_texts": (_int, [_u64, _i64, _i32, _i32, _vp, _i64, _vp]),
}
EXPORTS = tuple(_SIGNATURES)


class NativeError(RuntimeError):
    def __init__(self, code: int, what: str):
        super().__init__(f"libkllms_b200: {what} (code {code})")
        self.code = code


_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
    """dlopen the library and declare prototypes.  Raises if it is missing: no silent fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build the sm_90a library first (make -C k_llms_b200/csrc, or "
            "__graft_entry__.build()).  k_llms_b200 has no CPU fallback for the consensus hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        if restype is not ctypes.c_int:  # c_int is ctypes' default
            fn.restype = restype
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != KC_OK:
        raise NativeError(rc, load().kc_last_error().decode(errors="replace"))


def _require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("k_llms_b200 needs a CUDA (sm_90a) device: the consensus hot path has no CPU fallback")
    return torch


def _stream_ptr(torch, stream) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


def _bind(torch, t) -> None:
    check(load().kc_set_device(t.device.index if t.device.index is not None else torch.cuda.current_device()))


def vote(codes, none_code=None, stream=None) -> Tuple["torch.Tensor", "torch.Tensor"]:
    """K1 on device tensors.  codes: int32 [G, n] (cuda, contiguous); none_code: int32 [F] or None.
    Returns (win_code int32 [G], meta int32 [G] holding the packed uint32 word)."""
    torch = _require_cuda()
    assert codes.is_cuda and codes.dtype == torch.int32 and codes.dim() == 2 and codes.is_contiguous()
    G, n = codes.shape
    win = torch.empty(G, dtype=torch.int32, device=codes.device)
    meta = torch.empty(G, dtype=torch.int32, device=codes.device)
    nf = 0
    nc_ptr = None
    if none_code is not None:
        assert none_code.is_cuda and none_code.dtype == torch.int32 and none_code.is_contiguous()
        nf = none_code.numel()
        assert G % nf == 0, "n_groups must be a whole number of records"
        nc_ptr = none_code.data_ptr()
    _bind(torch, codes)
    check(load().kc_vote_i32(codes.data_ptr(), G, n, nc_ptr, nf, win.data_ptr(), meta.data_ptr(), _stream_ptr(torch, stream)))
    return win, meta


def vote_i8(codes, none_code=None, stream=None):
    """K1 on compact int8 cells (cuda int8 [G, n])."""
    torch = _require_cuda()
    assert codes.is_cuda and codes.dtype == torch.int8 and codes.dim() == 2 and codes.is_contiguous()
    G, n = codes.shape
    win = torch.empty(G, dtype=torch.int32, device=codes.device)
    meta = torch.empty(G, dtype=torch.int32, device=codes.device)
    nf, nc_ptr = 0, None
    if none_code is not None:
        nf, nc_ptr = none_code.numel(), none_code.data_ptr()
    _bind(torch, codes)
    check(load().kc_vote_i8(codes.data_ptr(), G, n, nc_ptr, nf, win.data_ptr(), meta.data_ptr(), _stream_ptr(torch, stream)))
    return win, meta


def numeric(vals, rel_eps: float = 0.03, abs_eps: float = 1e-6, stream=None):
    """K2 on device tensors.  vals: float64 [G, n].  Returns (value float64 [G], meta int32 [G])."""
    torch = _require_cuda()
    assert vals.is_cuda and vals.dtype == torch.float64 and vals.dim() == 2 and vals.is_contiguous()
    G, n = vals.shape
    value = torch.empty(G, dtype=torch.float64, device=vals.device)
    meta = torch.empty(G, dtype=torch.int32, device=vals.device)
    _bind(torch, vals)
    check(load().kc_numeric_f64(vals.data_ptr(), G, n, float(rel_eps), float(abs_eps), value.data_ptr(), meta.data_ptr(),
                                _stream_ptr(torch, stream)))
    return value, meta


def confidence(meta, numeric_kind: bool, pvf=None, stream=None):
    """Python-round(x,5)-exact confidences from result words.  meta int32 [G]; pvf float64 [G] or None."""
    torch = _require_cuda()
    assert meta.is_cuda and meta.dtype == torch.int32 and meta.is_contiguous()
    conf = torch.empty(meta.numel(), dtype=torch.float64, device=meta.device)
    pv = None
    if pvf is not None:
        assert pvf.is_cuda and pvf.dtype == torch.float64 and pvf.numel() == meta.numel() and pvf.is_contiguous()
        pv = pvf.data_ptr()
    _bind(torch, meta)
    check(load().kc_confidence_f64(meta.data_ptr(), meta.numel(), 1 if numeric_kind else 0, pv, conf.data_ptr(),
                                   _stream_ptr(torch, stream)))
    return conf


def logprob_sum(logprobs, offsets, stream=None):
    """K3: fp32 per-sequence sums.  logprobs float32 [T], offsets int64 [S+1] -> float32 [S]."""
    torch = _require_cuda()
    assert logprobs.is_cuda and logprobs.dtype == torch.float32 and offsets.dtype == torch.int64 and offsets.is_cuda
    out = torch.empty(offsets.numel() - 1, dtype=torch.float32, device=logprobs.device)
    _bind(torch, logprobs)
    check(load().kc_logprob_sum_f32(logprobs.data_ptr(), offsets.data_ptr(), out.numel(), out.data_ptr(),
                                    _stream_ptr(torch, stream)))
    return out


def weighted_vote(codes, seq_logprob, none_code=None, stream=None):
    """K3b: likelihood-weighted vote.  codes int32 [R, F, n], seq_logprob float32 [R, n] (cuda).
    Returns (win_code int32 [R*F], meta int32 [R*F], weight float32 [R*F])."""
    torch = _require_cuda()
    assert codes.is_cuda and codes.dtype == torch.int32 and codes.dim() == 3 and codes.is_contiguous()
    R, F, n = codes.shape
    assert seq_logprob.is_cuda and seq_logprob.dtype == torch.float32 and tuple(seq_logprob.shape) == (R, n)
    assert seq_logprob.is_contiguous()
    win = torch.empty(R * F, dtype=torch.int32, device=codes.device)
    meta = torch.empty(R * F, dtype=torch.int32, device=codes.device)
    weight = torch.empty(R * F, dtype=torch.float32, device=codes.device)
    nc = None
    if none_code is not None:
        assert none_code.is_cuda and none_code.dtype == torch.int32 and none_code.numel() == F
        nc = none_code.data_ptr()
    _bind(torch, codes)
    check(load().kc_weighted_vote_i32(codes.data_ptr(), seq_logprob.data_ptr(), R, F, n, nc, win.data_ptr(), meta.data_ptr(),
                                      weight.data_ptr(), _stream_ptr(torch, stream)))
    return win, meta, weight


def weighted_vote_groups(codes, group_record, seq_logprob, stream=None):
    """K3b over ragged records: codes int8 [G, n] (kc_vote_i8 cells), group_record int32 [G] (the record of each group),
    seq_logprob float32 [R, n] (cuda).  Returns (win_code int32 [G], meta int32 [G], weight float32 [G])."""
    torch = _require_cuda()
    assert codes.is_cuda and codes.dtype == torch.int8 and codes.dim() == 2 and codes.is_contiguous()
    G, n = codes.shape
    assert group_record.is_cuda and group_record.dtype == torch.int32 and group_record.is_contiguous() and group_record.numel() == G
    assert seq_logprob.is_cuda and seq_logprob.dtype == torch.float32 and seq_logprob.dim() == 2 and seq_logprob.is_contiguous()
    R = seq_logprob.shape[0]
    assert R == 0 or seq_logprob.shape[1] == n
    win = torch.empty(G, dtype=torch.int32, device=codes.device)
    meta = torch.empty(G, dtype=torch.int32, device=codes.device)
    weight = torch.empty(G, dtype=torch.float32, device=codes.device)
    _bind(torch, codes)
    check(load().kc_weighted_vote_groups_i8(codes.data_ptr(), G, n, group_record.data_ptr(), seq_logprob.data_ptr() if R else None, R,
                                            win.data_ptr(), meta.data_ptr(), weight.data_ptr(), _stream_ptr(torch, stream)))
    return win, meta, weight


def consensus_host(codes, none_code, vals, rel_eps=0.03, abs_eps=1e-6, device=0, out=None):
    """End-to-end entry with HOST numpy arrays (ideally backed by pinned memory).
    codes int32 [N, Fv, n] or None; none_code int32 [Fv] or None; vals float64 [N, Fx, n] or None.
    Returns dict(win_code, vote_meta, value, num_meta) of numpy arrays."""
    import numpy as np
    lib = load()
    N = n = Fv = Fx = 0
    if codes is not None:
        assert codes.dtype in (np.int32, np.int8) and codes.ndim == 3 and codes.flags.c_contiguous
        N, Fv, n = codes.shape
    if vals is not None:
        assert vals.dtype == np.float64 and vals.ndim == 3 and vals.flags.c_contiguous
        N2, Fx, n2 = vals.shape
        assert codes is None or (N2 == N and n2 == n)
        N, n = N2, n2
    out = out or {}
    win = out.get("win_code") if "win_code" in out else np.empty((N, Fv), dtype=np.int32)
    vmeta = out.get("vote_meta") if "vote_meta" in out else np.empty((N, Fv), dtype=np.uint32)
    value = out.get("value") if "value" in out else np.empty((N, Fx), dtype=np.float64)
    nmeta = out.get("num_meta") if "num_meta" in out else np.empty((N, Fx), dtype=np.uint32)
    if none_code is not None:
        none_code = np.ascontiguousarray(none_code, dtype=np.int32)
        assert none_code.size == Fv
    p = lambda a: a.ctypes.data if a is not None and a.size else None  # noqa: E731
    ms = ctypes.c_float(0.0)
    entry = lib.kc_consensus_host_i8 if (codes is not None and codes.dtype == np.int8) else lib.kc_consensus_host
    check(entry(p(codes), Fv, p(none_code), p(vals), Fx, N, n, float(rel_eps), float(abs_eps), p(win), p(vmeta),
                p(value), p(nmeta), device, ctypes.addressof(ms)))
    return {"win_code": win, "vote_meta": vmeta, "value": value, "num_meta": nmeta, "device_ms": float(ms.value)}


def numeric_medoid(cells, stream=None):
    """K5 on device tensors: the async dispatcher's numeric medoid.  cells float64 [G, n] (K2's encoding, n <= 64) ->
    (best int32 [G]: the medoid's position among the group's non-None cells, -1 for none; avg float64 [G]: its unrounded mean
    similarity, NaN with fewer than two non-None cells)."""
    torch = _require_cuda()
    assert cells.is_cuda and cells.dtype == torch.float64 and cells.dim() == 2 and cells.is_contiguous()
    G, n = cells.shape
    best = torch.empty(G, dtype=torch.int32, device=cells.device)
    avg = torch.empty(G, dtype=torch.float64, device=cells.device)
    _bind(torch, cells)
    check(load().kc_numeric_medoid_f64(cells.data_ptr(), G, n, best.data_ptr(), avg.data_ptr(), _stream_ptr(torch, stream)))
    return best, avg


SIM_METHODS = {"levenshtein": 0, "embeddings": 0, "jaccard": 1, "hamming": 2}  # "embeddings": pairs the planner sends here are Levenshtein pairs


def medoid_str(chars, str_off, grp_off, max_group=MAX_CANDIDATES, stream=None, method: str = "levenshtein"):
    """K4 on device tensors: chars uint8 [C], str_off int32 [S+1], grp_off int32 [G+1], max_group = largest group ->
    (best index int32 [G], mean similarity float64 [G]); method = the reference's string_similarity_method."""
    torch = _require_cuda()
    assert chars.is_cuda and chars.dtype == torch.uint8 and str_off.dtype == torch.int32 and grp_off.dtype == torch.int32
    G = grp_off.numel() - 1
    idx = torch.empty(G, dtype=torch.int32, device=chars.device)
    avg = torch.empty(G, dtype=torch.float64, device=chars.device)
    _bind(torch, chars)
    check(load().kc_medoid_str_method(chars.data_ptr(), str_off.data_ptr(), grp_off.data_ptr(), G, max(2, int(max_group)),
                                      SIM_METHODS[method], idx.data_ptr(), avg.data_ptr(), _stream_ptr(torch, stream)))
    return idx, avg


def _align_texts(values):
    """The candidate values of one record as ASCII JSON texts for kc_align_json(_batch), or None when the record needs the
    Python pre-pass."""
    import json
    # Precondition: the values look like json.loads output as far as OBJECT IDENTITY goes.  The reference's majority ordering
    # finds an aligned cell's source position by id() (majority_sorting.py:14-17), and the native code restates CPython's
    # behaviour for freshly parsed values (True / False / ints in [-5, 256] / one-character strings are shared objects,
    # everything else is distinct).  A list holding the SAME longer string / float / big int object twice (built in Python, or
    # deep-copied) breaks that: leave such records to the Python pre-pass, which sees the real identities.
    def shared_identity(v) -> bool:
        if isinstance(v, dict):
            return any(shared_identity(x) for x in v.values())
        if isinstance(v, list):
            seen = set()
            for x in v:
                if (isinstance(x, str) and len(x) > 1) or isinstance(x, float) or (isinstance(x, int) and not isinstance(x, bool) and not -5 <= x <= 256):
                    if id(x) in seen:
                        return True
                    seen.add(id(x))
            return any(shared_identity(x) for x in v)
        return False
    if any(shared_identity(v) for v in values):
        return None
    try:
        return [json.dumps(v).encode("ascii") for v in values]
    except (TypeError, ValueError):
        return None


def align_json(values, min_support_ratio: float):
    """H2: the alignment pre-pass (recursive_list_alignments, default similarity method) of ONE record in native code.
    values: n JSON-serialisable candidate values.  Returns the aligned values, or None when the record needs the Python
    pre-pass (long string pairs that go to the embeddings service, non-ASCII text, values json cannot carry)."""
    import json
    n = len(values)
    if n == 0:
        return None
    enc = _align_texts(values)
    if enc is None:
        return None
    texts = (ctypes.c_char_p * n)(*enc)
    out = (ctypes.c_char_p * n)()
    rc = load().kc_align_json(texts, None, n, float(min_support_ratio), out)
    if rc != 0:
        return None
    try:
        return [json.loads(out[i]) for i in range(n)]
    finally:
        load().kc_free_strings(out, n)


def align_json_batch(records, min_support_ratio: float = 0.51, device: int = 0, threads: int = 0, counts=None):
    """align_json for many records at once: the element similarities of their list fields are computed in one pass on
    `device` (kc_align_json_batch; device < 0 runs that pass on the host), the rest of the alignment on host threads.
    records: list of lists of candidate values.  Returns [align_json(r, min_support_ratio) for r in records] (None where a
    record needs the Python pre-pass).  counts (optional dict) receives "device_pairs" (element pairs the similarity pass
    decided) and "host_pairs" (pairs computed on the host while aligning)."""
    import json
    lib = load()
    res = [None] * len(records)
    by_n = {}  # one call per candidate count
    for i, values in enumerate(records):
        enc = _align_texts(values) if len(values) else None
        if enc is not None:
            by_n.setdefault(len(values), []).append((i, enc))
    total = [0, 0]
    for n, items in by_n.items():
        R = len(items)
        blobs = [b for _, enc in items for b in enc]
        texts = (ctypes.c_char_p * (R * n))(*blobs)
        lens = (ctypes.c_int64 * (R * n))(*[len(b) for b in blobs])
        out = (ctypes.c_void_p * (R * n))()
        status = (ctypes.c_int32 * R)()
        cnt = (ctypes.c_int64 * 2)()
        check(lib.kc_align_json_batch(ctypes.cast(texts, ctypes.c_void_p), ctypes.cast(lens, ctypes.c_void_p), R, n, float(min_support_ratio),
                                      int(device), int(threads), ctypes.cast(out, ctypes.c_void_p), ctypes.cast(status, ctypes.c_void_p),
                                      ctypes.cast(cnt, ctypes.c_void_p)))
        try:
            for k, (i, _) in enumerate(items):
                if status[k] == 0:
                    res[i] = [json.loads(ctypes.string_at(out[k * n + c])) for c in range(n)]
        finally:
            lib.kc_free_strings(ctypes.cast(out, ctypes.c_void_p), R * n)
        total[0] += cnt[0]
        total[1] += cnt[1]
    if counts is not None:
        counts["device_pairs"], counts["host_pairs"] = total
    return res


def levenshtein(a: str, b: str) -> int:
    """Edit distance through the native library (code points must be Latin-1; callers pass normalised ASCII)."""
    ba, bb = a.encode("latin-1"), b.encode("latin-1")
    return int(load().kc_levenshtein(ba, len(ba), bb, len(bb)))


def consolidate_json(records, rel_eps: float = 0.03, abs_eps: float = 1e-6, device: int = 0, threads: int = 0):
    """H1: native consolidation of records of scalars, nested objects and lists (default settings).  records: list of lists of n candidate content strings.
    Returns a list of (content_str, likelihoods_json_str) or None where the record needs the Python path."""
    lib = load()
    R = len(records)
    if R == 0:
        return []
    n = len(records[0])
    assert all(len(r) == n for r in records), "every record needs the same number of candidates"
    blobs = [t.encode("utf-8") for r in records for t in r]
    texts = (ctypes.c_char_p * (R * n))(*blobs)
    lens = (ctypes.c_int64 * (R * n))(*[len(b) for b in blobs])
    out_c = (ctypes.c_void_p * R)()
    out_l = (ctypes.c_void_p * R)()
    status = (ctypes.c_uint8 * R)()
    check(lib.kc_consolidate_json(ctypes.cast(texts, ctypes.c_void_p), ctypes.cast(lens, ctypes.c_void_p), R, n, float(rel_eps),
                                  float(abs_eps), device, threads, ctypes.cast(out_c, ctypes.c_void_p),
                                  ctypes.cast(out_l, ctypes.c_void_p), ctypes.cast(status, ctypes.c_void_p)))
    res = []
    for i in range(R):
        if status[i] == 0:
            res.append((ctypes.string_at(out_c[i]).decode("ascii"), ctypes.string_at(out_l[i]).decode("ascii")))
        else:
            res.append(None)
    lib.kc_free_strings(ctypes.cast(out_c, ctypes.c_void_p), R)
    lib.kc_free_strings(ctypes.cast(out_l, ctypes.c_void_p), R)
    return res


def pinned_empty(shape, dtype):
    """numpy array backed by page-locked memory from kc_host_alloc (freed when the array is collected)."""
    import numpy as np
    lib = load()
    dt = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dt.itemsize
    ptr = lib.kc_host_alloc(max(nbytes, 1))
    if not ptr:
        raise MemoryError(f"kc_host_alloc({nbytes}) failed")
    buf = (ctypes.c_uint8 * max(nbytes, 1)).from_address(ptr)
    arr = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
    import weakref
    weakref.finalize(buf, lib.kc_host_free, ptr)
    return arr


class JsonStats(ctypes.Structure):
    """kc_json_stats (include/kllms_b200.h)."""
    _fields_ = [(k, ctypes.c_int64) for k in ("n_records", "n_device", "n_host", "n_python", "input_bytes", "output_bytes")] + \
               [("chunks", ctypes.c_int32), ("streams", ctypes.c_int32)] + \
               [(k, ctypes.c_double) for k in ("h2d_ms", "plan_ms", "kernel_ms", "emit_ms", "d2h_ms", "device_path_wall_ms",
                                               "host_path_wall_ms", "wall_ms")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


JSON_DEVICE_ONLY = 1
JSON_NUMERIC_MEDOID = 2  # the async dispatcher: numeric fields are similarity medoids (K5); implies JSON_DEVICE_ONLY
JSON_KEY_UNION = 4  # candidates that differ in shape (key order, missing / extra keys, null sub-objects) stay on the device
JSON_LISTS = 8  # records with list fields stay on the device: aligned by H2 on host threads, consolidated in a list round
JSON_UNICODE = 16  # similarity-medoid fields with non-ASCII text or \uXXXX escapes stay on the device (vote fields decline)


def pack_texts(records, pinned: bool = True):
    """records: list of lists of n candidate content strings -> (blob uint8 array, off int64 array [R*n+1], n): the packed
    form kc_consolidate_json_packed takes (blob in page-locked memory when `pinned`)."""
    import numpy as np
    R = len(records)
    n = len(records[0]) if R else 0
    assert all(len(r) == n for r in records), "every record needs the same number of candidates"
    enc = [t.encode("utf-8") for r in records for t in r]
    off = np.zeros(R * n + 1, dtype=np.int64)
    if enc:
        np.cumsum(np.fromiter((len(b) for b in enc), dtype=np.int64, count=len(enc)), out=off[1:])
    total = int(off[-1])
    blob = pinned_empty((max(total, 1),), np.uint8) if pinned else np.empty(max(total, 1), dtype=np.uint8)
    if total:
        blob[:total] = np.frombuffer(b"".join(enc), dtype=np.uint8)
    return blob, off, n


class PackedResult:
    """View of a kc_json_result: `content(r)` / `likelihoods(r)` are the texts of record r (None when status is 1)."""

    def __init__(self, handle, R):
        import numpy as np
        self._h, self.R = handle, R
        lib = load()
        ptrs = [ctypes.c_void_p() for _ in range(7)]
        self.stats = JsonStats()
        check(lib.kc_json_result_view(handle, *[ctypes.byref(p) for p in ptrs], ctypes.addressof(self.stats)))
        as_i64 = lambda p: np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_int64)), shape=(R,)) if R else np.zeros(0, np.int64)  # noqa: E731
        as_u8 = lambda p: np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_uint8)), shape=(R,)) if R else np.zeros(0, np.uint8)  # noqa: E731
        self._text = ptrs[0].value or 0
        self.c_off, self.c_len, self.l_off, self.l_len = as_i64(ptrs[1]), as_i64(ptrs[2]), as_i64(ptrs[3]), as_i64(ptrs[4])
        self.status, self.why = as_u8(ptrs[5]), as_u8(ptrs[6])

    def content(self, r):
        return None if self.status[r] == 1 else ctypes.string_at(self._text + int(self.c_off[r]), int(self.c_len[r])).decode("ascii")

    def likelihoods(self, r):
        return None if self.status[r] == 1 else ctypes.string_at(self._text + int(self.l_off[r]), int(self.l_len[r])).decode("ascii")

    def pairs(self):
        return [None if self.status[r] == 1 else (self.content(r), self.likelihoods(r)) for r in range(self.R)]

    def close(self):
        if self._h is not None:
            load().kc_json_result_free(self._h)
            self._h = None

    def __del__(self):
        self.close()


def consolidate_json_packed(blob, off, n, rel_eps: float = 0.03, abs_eps: float = 1e-6, device: int = 0, threads: int = 0,
                            flags: int = 0) -> PackedResult:
    """H1g: the JSON-in / JSON-out consolidation with the JSON work on the device (kc_consolidate_json_packed).
    blob uint8 array of all candidate texts, off int64 [R*n+1]; see pack_texts()."""
    lib = load()
    R = (len(off) - 1) // n if n else 0
    h = ctypes.c_void_p()
    check(lib.kc_consolidate_json_packed(blob.ctypes.data, off.ctypes.data, R, n, float(rel_eps), float(abs_eps), device, threads,
                                         flags, ctypes.byref(h)))
    return PackedResult(h, R)


def consolidate_json_packed_weighted(blob, off, n, seq_logprob, rel_eps: float = 0.03, abs_eps: float = 1e-6, device: int = 0,
                                     threads: int = 0, flags: int = 0) -> PackedResult:
    """H1g with likelihood-weighted vote leaves (kc_consolidate_json_packed_weighted, DESIGN.md §5): seq_logprob float32
    [R*n] = the candidates' sequence logprobs, record-major.  Records the device path declines keep status 1 (no host path)."""
    import numpy as np
    lib = load()
    R = (len(off) - 1) // n if n else 0
    seq = np.ascontiguousarray(seq_logprob, dtype=np.float32).reshape(-1)
    assert seq.size == R * n, "one sequence logprob per candidate"
    h = ctypes.c_void_p()
    check(lib.kc_consolidate_json_packed_weighted(blob.ctypes.data, off.ctypes.data, seq.ctypes.data if seq.size else None, R, n,
                                                  float(rel_eps), float(abs_eps), device, threads, flags, ctypes.byref(h)))
    return PackedResult(h, R)


def s32_texts_packed(n_records: int, n: int, seed: int, pinned: bool = True, threads: int = 0):
    """Schema S32 (SURVEY.md §8d) as candidate TEXTS in packed form (blob uint8, off int64 [R*n+1]), generated natively
    (kc_debug_s32_texts: exactly json.dumps' formatting; tests/test_jsongpu_host_logic.py checks that)."""
    import numpy as np
    lib = load()
    off = np.zeros(n_records * n + 1, dtype=np.int64)
    check(lib.kc_debug_s32_texts(seed, n_records, n, threads, None, 0, off.ctypes.data))
    total = int(off[-1])
    blob = pinned_empty((max(total, 1),), np.uint8) if pinned else np.empty(max(total, 1), dtype=np.uint8)
    check(lib.kc_debug_s32_texts(seed, n_records, n, threads, blob.ctypes.data, total, off.ctypes.data))
    return blob, off
