"""GPU: every K1 kernel (kc_vote.cuh) on the vote's decision edges, against the brute force of tests/test_vote_edges_host.py
(every class counted, no guess, no early stop) and the C oracle.

The families (exact ties in every first-seen order with a tied class starting at lanes 0, 31, 32, 63; the guess's class at
exactly half of the voters or one more; guesses fooled into an absent code, a present minority or a negative value, and at
n = 64 into the right code from cells that do not hold it; the scan reaching a last class of best_cnt - 1, best_cnt or
best_cnt + 1 cells; codes at the ends of int32 and int8; None and absent mixtures) go through kc_vote_i32 without and with a
none_code table of 1, 3, 7 and 33 fields at every n that picks another kernel or padding, through kc_vote_i8 on the rows
that fit int8 cells, and through one non-local route.  Group counts are not multiples of the multi-group kernels' unit, so
their tails (one launch per group with a none_code table) run too.  Each test checks under torch.profiler that the kernels
it means to test ran, and counts on the host how many groups reach the scan's hard cases, so that a generator change cannot
quietly make the cases easy."""
import json
import random

import numpy as np
import pytest

from oracle import columnar as OC
from tests import test_vote_edges_host as H
from tests.helpers import assert_kernels_ran, profiled

pytestmark = pytest.mark.gpu

N_LIST = H.N_LIST
F_LIST = [None, 1, 3, 7, 33]  # None: no none_code table
PER_FAMILY = 167  # rows per family and table: 1002 groups, not a multiple of 8, 3, 7 or 33
MANY = {32: 400_003, 64: 160_001}  # over three waves of the TMA kernels' persistent grid on an H100 (132 SMs)


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _nc(has_nc):
    return "true" if has_nc else "false"


def i32_kernels(n, has_nc, G, local=True):
    """The kernels kc_vote_i32 (local, or a non-local route) launches for G groups of n cells (test_gpu_routes.COVERAGE)."""
    nc = _nc(has_nc)
    if n in (2, 4, 8):
        direct = f"vote_direct_kernel<int,{n},true,{nc},{'true' if n >= 4 else 'false'}>"
        if not local:
            return [direct]
        gpt = 16 // n
        return [f"vote_multi_kernel<{n},{gpt},{nc}>"] + ([direct] if G % gpt else [])
    if n in (1, 16):
        return [f"vote_direct_kernel<int,{n},true,{nc},{'true' if n == 16 else 'false'}>"]
    if n in (32, 64):
        return [f"vote_tma_kernel<{n},{8 if n == 32 else 4},2,{nc}>"]
    return [f"vote_direct_kernel<int,{max(4, H.pow2(n))},false,{nc},false>"]


def i8_kernels(n, has_nc):
    np_ = max(4, H.pow2(n))
    return [f"vote_direct_kernel<signedchar,{np_},{'true' if n == np_ else 'false'},{_nc(has_nc)},false>"]


def run_i32(abi, codes, table):
    from tests.test_gpu_routes import vote_local
    w, m = vote_local(abi, codes, table)
    return w.cpu().numpy(), m.cpu().numpy().view(np.uint32)


def run_i8(codes, table):
    torch = _torch()
    from k_llms_b200 import _native as K
    w, m = K.vote_i8(torch.from_numpy(codes.astype(np.int8)).cuda(), torch.from_numpy(table).cuda() if table is not None else None)
    return w.cpu().numpy(), m.cpu().numpy().view(np.uint32)


def _table(n, F, wide):
    return H.nc_table(random.Random(7 * n + (F or 0) + 1000 * wide), F, wide) if F else None


# floors over the ten cases of one n (five tables, int32-wide and int8-narrow codes), counted on the host
SCAN_FLOOR = 3000   # groups without an absent cell that the guess leaves to the scan (n a power of two from 2 on)
TIE_FLOOR = 1500    # groups with TIE (n >= 2)
EDGE_FLOOR = 1200   # scans that finish a class with remaining == best_cnt (n >= 2; n a power of two: without absent cells)
HIGH_FLOOR = 500    # n = 64: winners whose first cell is 32 or more


@pytest.mark.parametrize("n", N_LIST)
def test_every_k1_kernel_on_the_edge_families(n):
    torch = _torch()
    from tests.test_gpu_routes import Abi, check_vote_route
    abi = Abi()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    expected, total = set(), {}
    with profiled() as prof:
        for wide in (True, False):
            for F in F_LIST:
                table = _table(n, F, wide)
                codes, _, ncg = H.family_rows(9000 + 31 * n + (F or 0) + 500 * wide, n, PER_FAMILY, table, wide)
                what = (n, F, "int32" if wide else "int8")
                ref = H.brute(codes, ncg)
                ew, em = OC.vote(codes, table)
                H.check_against(ew, em, ref, ("C oracle",) + what)
                H.check_against(*run_i32(abi, codes, table), ref, ("kc_vote_i32",) + what)
                expected.update(i32_kernels(n, F is not None, len(codes)))
                if not wide:
                    H.check_against(*run_i8(codes, table), ref, ("kc_vote_i8",) + what)
                    expected.update(i8_kernels(n, F is not None))
                else:  # the non-local route: n = 2, 4, 8 through vote_direct_kernel's vote_core, not vote_core_small
                    check_vote_route(abi, "peers1", codes, table, flag, what)
                    expected.update(i32_kernels(n, F is not None, len(codes), local=False))
                for k, v in H.counts(codes, ncg, ref).items():
                    total[k] = total.get(k, 0) + v
    assert_kernels_ran(prof, expected)
    print(f"\nn={n}: {total}; kernels {sorted(expected)}")
    if n >= 2:
        assert total["TIE"] >= TIE_FLOOR, total
    if n >= 2 and n == H.pow2(n):
        assert total["scan, no absent cell"] >= SCAN_FLOOR, total
        assert total["... no absent cell"] >= EDGE_FLOOR, total
    elif n >= 2:
        assert total["scan at remaining == best"] >= EDGE_FLOOR, total
    if n == 64:
        assert total["first index >= 32"] >= HIGH_FLOOR, total


@pytest.mark.parametrize("n", [32, 64])
def test_tma_kernels_over_many_waves(n):
    """The n = 32 and n = 64 families tiled past three waves of the persistent TMA grid with a 7-field none_code table: every
    group against the C oracle, a sample against the brute force."""
    _torch()
    from tests.test_gpu_routes import Abi
    table = _table(n, 7, True)
    codes, _, _ = H.family_rows(77 + n, n, 7 * 120, table, True)  # 7 * 720 rows: whole records, so tiling keeps the fields
    reps = -(-MANY[n] // len(codes))
    big = np.ascontiguousarray(np.tile(codes, (reps, 1))[:MANY[n]])
    with profiled() as prof:
        win, meta = run_i32(Abi(), big, table)
    assert_kernels_ran(prof, i32_kernels(n, True, len(big)))
    ew, em = OC.vote(big, table)
    H.check_against(win, meta, dict(win=ew.astype(np.int64), meta=em), ("C oracle, all groups", n))
    pick = np.random.default_rng(n).choice(len(big), 40_000, replace=False)
    ref = H.brute(big[pick], table[pick % 7])
    H.check_against(win[pick], meta[pick], ref, ("brute force, sample", n))


def json_records(n, R, seed):
    """R records of n candidates whose string ("s"), enum ("e") and bool ("b") fields are rows of families 1 (ties), 2 (the
    majority boundary) and 6 (None / absent mixtures): a code c is "w<c>", "E<c>" or c odd; None is null (a bool's None
    votes False).  Absent cells are spelled null too: a key missing from some candidates sends most records to the host."""
    rows = {}
    for key, nc in (("s", -1), ("e", -1), ("b", 0)):
        r = random.Random(seed + ord(key))
        fam = [(1, 2, 6)[i % 3] for i in range(R)]
        rows[key] = [H.MAKERS[f](r, n, nc, False) for f in fam]
    spell = {"s": lambda c: f"w{c}", "e": lambda c: f"E{c}", "b": lambda c: c % 2 == 1}
    records = []
    for i in range(R):
        texts = []
        for j in range(n):
            obj = {}
            for key in ("s", "e", "b"):
                c = rows[key][i][j]
                obj[key] = spell[key](c) if c >= 0 else None
            texts.append(json.dumps(obj))
        records.append(texts)
    return records


@pytest.mark.parametrize("n", [3, 8, 32])
def test_device_json_path_on_the_edge_families(n):
    """Records built from families 1, 2 and 6 through kc_consolidate_json_packed (K1 on int8 cells through kc_vote_i8, with
    the bool field's none_code): value and likelihoods byte for byte against the reference's client order."""
    _torch()
    from k_llms_b200 import _native as K
    from tests.test_gpu_json import _expected
    records = json_records(n, 450, 40 + n)
    blob, off, _ = K.pack_texts(records)
    res = K.consolidate_json_packed(blob, off, n)
    try:
        on_device = 0
        for r, texts in enumerate(records):
            if res.status[r] == 1:
                continue
            on_device += res.status[r] == 0
            assert (res.content(r), res.likelihoods(r)) == _expected(texts), (r, texts, res.status[r])
        assert on_device >= 0.9 * len(records), (on_device, len(records))
    finally:
        res.close()
