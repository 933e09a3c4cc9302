"""The multi-GPU wire words (k_llms_b200/distributed.py, csrc/kc_push.cuh) on the CPU: every valid result word that fits the
narrow (u16) or the wide (u32) words, packed with wire_pack_votes / wire_pack_num and decoded with wire_confidences, gives
back the winning code and exactly the confidences the reference computes with Python's round(x, 5) from the full word."""
import numpy as np
import pytest

from k_llms_b200.distributed import wire_confidences, wire_pack_num, wire_pack_votes

HAS_VALUE, SINGLE, TIE, NO_FINITE = 1, 2, 4, 8


def result_word(idx, support, nn, present, flags):
    return (idx & 0x3F) | (support << 6) | (nn << 13) | (present << 20) | (flags << 27)


def triples(max_present):
    """Every (support, nn, present) with support <= nn <= present <= max_present, as three int64 arrays."""
    t = np.array([(s, nn, p) for p in range(max_present + 1) for nn in range(p + 1) for s in range(nn + 1)], dtype=np.int64)
    return t[:, 0], t[:, 1], t[:, 2]


def ratio_table(max_present, fn):
    """fn(a, b) for every 0 <= a <= b <= max_present, b >= 1, looked up as table[a, b]."""
    t = np.zeros((max_present + 1, max_present + 1))
    for b in range(1, max_present + 1):
        for a in range(b + 1):
            t[a, b] = fn(a, b)
    return t


def vote_words(max_present, codes):
    """Every K1 result word with present <= max_present: a value (support >= 1, with and without the tie flag, each winning
    code in `codes`) or none (support 0, winning code -1).  Returns (win, meta, expected confidence)."""
    support, nn, present = triples(max_present)
    r5 = ratio_table(max_present, lambda a, b: round(a / b, 5))
    win, meta, conf = [], [], []
    none = support == 0
    win.append(np.full(none.sum(), -1))
    meta.append(result_word(0, 0, nn[none], present[none], 0))
    conf.append(np.where(present[none] == 0, 1.0, 0.0))
    s, v, p = support[~none], nn[~none], present[~none]
    for code in codes:
        for flags in (HAS_VALUE, HAS_VALUE | TIE):
            win.append(np.full(s.size, code))
            meta.append(result_word(p - 1, s, v, p, flags))
            conf.append(r5[s, p])
    return (np.concatenate(win).astype(np.int32), np.concatenate(meta).astype(np.uint32), np.concatenate(conf))


def numeric_words(max_present):
    """Every K2 result word with present <= max_present under the flag combinations of
    test_gpu_kernels.py::test_confidence_matches_python_round, with the confidences it expects at pvf = 1."""
    support, nn, present = triples(max_present)
    r5 = ratio_table(max_present, lambda a, b: round(a / b, 5))
    inv = ratio_table(max_present, lambda a, b: 1 / b)
    frac = ratio_table(max_present, lambda a, b: a / b)
    meta, conf = [], []
    for f in (HAS_VALUE, HAS_VALUE | SINGLE, NO_FINITE, 0):
        keep = (support > 0) & (present > 0) if f & (HAS_VALUE | NO_FINITE) else np.ones(support.size, dtype=bool)
        s, v, p = support[keep], nn[keep], present[keep]
        meta.append(result_word(0, s, v, p, f))
        if f & HAS_VALUE:
            conf.append(inv[0, p] if f & SINGLE else r5[s, v])
        elif f & NO_FINITE:
            conf.append(frac[v, p])
        else:
            conf.append(np.where(p == 0, 1.0, 0.0))
    return np.concatenate(meta).astype(np.uint32), np.concatenate(conf)


@pytest.mark.parametrize("wide", [False, True], ids=["narrow", "wide"])
def test_wire_words_decode_to_python_round_confidences(wide):
    max_present = 64 if wide else 31
    code_max = (1 << 18) - 1 if wide else 63
    win, vmeta, exp_vconf = vote_words(max_present, (0, 1, code_max - 1, code_max))
    nmeta, exp_nconf = numeric_words(max_present)
    vw, nw = wire_pack_votes(win, vmeta, wide), wire_pack_num(nmeta, wide)
    assert vw.dtype == (np.uint32 if wide else np.uint16) and nw.dtype == vw.dtype
    vconf, _ = wire_confidences(vw, np.zeros(0, dtype=vw.dtype), wide)
    _, nconf = wire_confidences(np.zeros(0, dtype=vw.dtype), nw, wide)
    has = ((vmeta >> 6) & 0x7F) > 0
    assert np.array_equal((vw.astype(np.uint32) & code_max)[has], win[has].astype(np.uint32))
    bad = np.nonzero(vconf != exp_vconf)[0]
    assert bad.size == 0, [(hex(vmeta[i]), vconf[i], exp_vconf[i]) for i in bad[:5]]
    bad = np.nonzero(nconf != exp_nconf)[0]
    assert bad.size == 0, [(hex(nmeta[i]), nconf[i], exp_nconf[i]) for i in bad[:5]]


def test_wire_words_cover_the_field_limits():
    """The enumeration above reaches the largest present / support / code each word holds."""
    for wide, max_present, code_max in ((False, 31, 63), (True, 64, (1 << 18) - 1)):
        win, vmeta, _ = vote_words(max_present, (0, code_max))
        vw = wire_pack_votes(win, vmeta, wide).astype(np.uint32)
        s_shift, p_shift, mask = (18, 25, 0x7F) if wide else (6, 11, 31)
        assert ((vw >> s_shift) & mask).max() == max_present and ((vw >> p_shift) & mask).max() == max_present
        assert (vw & code_max).max() == code_max
