"""The device JSON path's phases with KC_JSON_KEY_UNION, instantiated on the host: kc_debug_jsongpu_plan_flags -> the C oracle in
K1's place (or K3b's, with candidate sums), K2's (or numpy's medoid in K5's, numeric_medoid) and K4's -> kc_debug_jsongpu_emit_weighted."""
import ctypes as c

import numpy as np

from oracle import columnar as OC
from tests.async_native_oracle import numeric_medoid as k5_oracle


def jsongpu_union_with_oracle(records, seq=None, numeric_medoid=False):
    """Returns (pairs, status): pairs[r] = (content, likelihoods) or None where the device path declines the record (status[r] =
    its reason code).  seq: float32 [R*n] candidate sums (likelihood-weighted votes); numeric_medoid: KC_JSON_NUMERIC_MEDOID."""
    from k_llms_b200 import _native as K
    lib = K.load()
    R = len(records)
    if R == 0:
        return [], []
    blob, off, n = K.pack_texts(records, pinned=False)
    flags = K.JSON_KEY_UNION | (K.JSON_NUMERIC_MEDOID if numeric_medoid else 0)
    h = c.c_void_p()
    K.check(lib.kc_debug_jsongpu_plan_flags(blob.ctypes.data, off.ctypes.data, R, n, flags, c.byref(h)))
    try:
        vc, nc, st, gr = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        gv, gx = c.c_int64(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_inputs(h, c.byref(vc), c.byref(gv), c.byref(nc), c.byref(gx), c.byref(st)))
        K.check(lib.kc_debug_jsongpu_group_records(h, c.byref(gr)))
        vmeta, vweight = np.zeros(max(gv.value, 1), dtype=np.uint32), np.zeros(max(gv.value, 1), dtype=np.float32)
        if gv.value:
            codes = np.ctypeslib.as_array(c.cast(vc, c.POINTER(c.c_int8)), shape=(gv.value, n)).astype(np.int32)
            if seq is None:
                _, vmeta = OC.vote(codes, None)
            else:
                rec = np.ctypeslib.as_array(c.cast(gr, c.POINTER(c.c_int32)), shape=(gv.value,)).copy()
                _, vmeta, vweight = OC.weighted_vote(codes[:, None, :], np.asarray(seq, dtype=np.float32).reshape(R, n)[rec])
        nvalue, nmeta = np.zeros(max(gx.value, 1), dtype=np.float64), np.zeros(max(gx.value, 1), dtype=np.uint32)
        best, avg = np.zeros(max(gx.value, 1), dtype=np.int32), np.zeros(max(gx.value, 1), dtype=np.float64)
        if gx.value:
            cells = np.ctypeslib.as_array(c.cast(nc, c.POINTER(c.c_double)), shape=(gx.value, n)).copy()
            if numeric_medoid:
                best, avg = k5_oracle(cells)
            else:
                nvalue, nmeta = OC.numeric(cells)
        K.check(lib.kc_debug_jsongpu_set_numeric_medoid(h, best.ctypes.data, avg.ctypes.data))
        mc, so, go, gm = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_int64()
        K.check(lib.kc_debug_jsongpu_medoid_inputs(h, c.byref(mc), c.byref(so), c.byref(go), c.byref(gm)))
        midx, mavg = np.zeros(max(gm.value, 1), dtype=np.int32), np.zeros(max(gm.value, 1), dtype=np.float64)
        if gm.value:
            OC.lib().ko_medoid_str(mc, so, go, gm.value, midx.ctypes.data, mavg.ctypes.data)
        K.check(lib.kc_debug_jsongpu_set_medoid(h, midx.ctypes.data, mavg.ctypes.data))
        pc, po, pl, plo = c.c_void_p(), c.c_void_p(), c.c_void_p(), c.c_void_p()
        K.check(lib.kc_debug_jsongpu_emit_weighted(h, vmeta.ctypes.data, vweight.ctypes.data if seq is not None else None,
                                                   nvalue.ctypes.data, nmeta.ctypes.data, c.byref(pc), c.byref(po), c.byref(pl),
                                                   c.byref(plo)))
        status = np.ctypeslib.as_array(c.cast(st, c.POINTER(c.c_uint8)), shape=(R,)).copy()
        co = np.ctypeslib.as_array(c.cast(po, c.POINTER(c.c_int64)), shape=(R + 1,))
        lo = np.ctypeslib.as_array(c.cast(plo, c.POINTER(c.c_int64)), shape=(R + 1,))
        pairs = [None if status[r] else (c.string_at(pc.value + int(co[r]), int(co[r + 1] - co[r])).decode("ascii"),
                                         c.string_at(pl.value + int(lo[r]), int(lo[r + 1] - lo[r])).decode("ascii")) for r in range(R)]
        return pairs, [int(s) for s in status]
    finally:
        lib.kc_debug_jsongpu_free(h)
