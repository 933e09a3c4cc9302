"""GPU: K4 under Levenshtein (kc_medoid.cuh, medoid_kernel<4>) on the edge families of tests/test_medoid_edges_host.py, against
the brute force there (a numpy Levenshtein DP, np.nanmean over the matrix with a NaN diagonal, np.argmax) and the C oracle.

The families (patterns of 1 to 64 characters against texts of up to 2000 in styles that reach every carry and the top bit;
equal-length pairs and a long string at index 0, 31, 32 or 63 of 64; empty strings and similarities at the 1e-8 floor; u = 1,
33 and 64 classes, late duplicates, an FNV-1a collision on both sides of k = 32; exact ties within a lane and across lanes;
groups whose winner numpy's summation order decides) run through kc_medoid_str_method at every max_group they fit, through
kc_medoid_str_host, over about six waves of the persistent grid, as multi-word string fields through the device JSON path and
H1, and as list nodes through the alignment pre-pass's similarity kernel.  Index and mean must match bit for bit."""
import json

import numpy as np
import pytest

from k_llms_b200 import _native as K
from oracle import columnar as OC
from tests import test_medoid_edges_host as H
from tests.alignsim_cases import assert_matrices
from tests.helpers import assert_kernels_ran, consolidate_json_with_oracle, jsongpu_with_oracle, profiled

pytestmark = pytest.mark.gpu

MAX_GROUPS = (2, 5, 32, 33, 64)
KERNEL = "medoid_kernel<4>"
MANY = 3300  # at max_group = 64 one 4-warp CTA fits an SM: about six waves of a 132-SM H100's 528 warps


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def run_device(groups, max_group):
    torch = _torch()
    chars, so, go = OC.pack_string_groups(groups)
    idx, avg = K.medoid_str(torch.from_numpy(chars).cuda(), torch.from_numpy(so).cuda(), torch.from_numpy(go).cuda(), max_group=max_group)
    return idx.cpu().numpy(), avg.cpu().numpy()


def run_host_entry(groups, max_group):
    """kc_medoid_str_host: host buffers in, the same kernel on device 0, host buffers out."""
    chars, so, go = OC.pack_string_groups(groups)
    idx, avg = np.zeros(len(groups), np.int32), np.zeros(len(groups))
    K.check(K.load().kc_medoid_str_host(chars.ctypes.data, int(so[-1]), so.ctypes.data, go.ctypes.data, len(groups), max_group,
                                        idx.ctypes.data, avg.ctypes.data, 0))
    return idx, avg


def check(got, exp, what):
    (gi, ga), (ei, ea) = got, exp
    bad = np.flatnonzero((np.asarray(gi) != ei) | (np.asarray(ga).view(np.uint64) != ea.view(np.uint64)))
    assert not bad.size, (what, bad.size, bad[:5], gi[bad[:3]], ga[bad[:3]], ei[bad[:3]], ea[bad[:3]])


@pytest.mark.parametrize("max_group", MAX_GROUPS)
def test_k4_on_the_edge_families(max_group):
    """Every family group of at most max_group strings through kc_medoid_str_method and kc_medoid_str_host: the brute
    force's index and mean bits, and the C oracle's."""
    _torch()
    per_family = {f: [g for g in H.families()[f] if len(g) <= max_group] for f in H.FAMILIES}
    groups = [g for f in H.FAMILIES for g in per_family[f]]
    exp = H.brute(groups)
    check(OC.medoid(groups), exp, ("C oracle", max_group))
    with profiled() as prof:
        dev = run_device(groups, max_group)
    assert_kernels_ran(prof, [KERNEL])
    host = run_host_entry(groups, max_group)
    check(dev, exp, ("kc_medoid_str_method", max_group))
    check(host, exp, ("kc_medoid_str_host", max_group))
    sizes = {f: len(v) for f, v in per_family.items()}
    print(f"\nmax_group={max_group}: {len(groups)} groups {sizes}")
    assert len(groups) >= {2: 20, 5: 60, 32: 200, 33: 220, 64: 400}[max_group], sizes


def test_k4_over_many_waves():
    """The families shuffled and tiled to over 3,000 groups at max_group = 64: every warp of the persistent grid takes
    several groups of different u through the same shared memory."""
    groups = H.all_groups()
    exp_i, exp_a = H.brute(groups)
    order = np.random.default_rng(4).permutation(np.tile(np.arange(len(groups)), -(-MANY // len(groups))))[:MANY]
    big = [groups[i] for i in order]
    with profiled() as prof:
        dev = run_device(big, 64)
    assert_kernels_ran(prof, [KERNEL])
    check(dev, (exp_i[order], exp_a[order]), "many waves")
    check(run_host_entry(big, 64), (exp_i[order], exp_a[order]), "many waves, kc_medoid_str_host")


def test_json_paths_on_the_edge_groups():
    """The edge groups as multi-word string fields (patterns of 31, 32, 33, 49 and 50 characters against one string longer
    than 50): the device JSON path takes every record, prints what its host instantiation with the C oracle prints and the
    brute force's medoid string; H1 prints what it prints with the C oracle in K4's place.  Under JSON_DEVICE_ONLY a
    record the device path does not decide itself comes back declined, so status 0 means K4 on the device chose its
    medoid.  No profiler session here: the JSON paths launch from library threads, and the kernel checks above stay on
    plain launches."""
    _torch()
    total = 0
    for n, (records, groups) in sorted(H.json_records(H.json_groups()).items()):
        idx, _ = H.brute(groups)
        blob, off, _ = K.pack_texts(records)
        res = K.consolidate_json_packed(blob, off, n, flags=K.JSON_DEVICE_ONLY)
        try:
            got, status = res.pairs(), list(res.status)
        finally:
            res.close()
        host, host_status = jsongpu_with_oracle(records)
        h1, h1_oracle = K.consolidate_json(records), consolidate_json_with_oracle(records)
        for r, texts in enumerate(records):
            want = json.loads(texts[idx[r]])["s"]
            assert status[r] == 0 and host_status[r] == 0 and got[r] == host[r], (n, r, status[r], got[r], host[r])
            assert json.loads(got[r][0])["s"] == want, (n, r, got[r], want)
            assert h1[r] is not None and h1[r] == h1_oracle[r], (n, r, h1[r], h1_oracle[r])
            total += 1
    assert total >= 200, total


def test_alignsim_kernel_on_the_edge_nodes():
    """alignsim_kernel on list nodes with patterns of 31, 32, 33, 49 and 50 characters against texts of up to 2000: every
    decided pair equals 1 - d / longest (floored) and the host instantiation's bits; NaN on the diagonal and between two
    strings longer than 50 characters."""
    _torch()
    nodes = [nd for seed in (0, 1, 2) for nd in H.align_nodes(seed)]
    exp = H.align_expected(nodes)
    got = H.run_align(nodes, device=0)
    assert_matrices(got, exp)
    assert_matrices(got, H.run_align(nodes, -1, 32))
