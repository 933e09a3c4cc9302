"""CPU checks of what the GPU instantiations of shared host/device code read or do differently from the host ones:
the device copies of the Ryu power-of-5 tables (float.__repr__ on the device reads kPow5*Dev, the host kPow5*Host), and
the element-similarity pass (kc_alignsim.cuh) walking each node's pairs over 32 lanes as a warp does."""
import os
import random
import re

import numpy as np

from tests.alignsim_cases import NODE_SIZES, assert_matrices, expected_matrices, node_sets, run_nodes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tables():
    text = open(os.path.join(ROOT, "k_llms_b200", "csrc", "kc_ryu_tables.cuh")).read()
    found = {}
    for m in re.finditer(r"static (?:__device__ )?const uint64_t (\w+)\[(\d+)\]\[2\] = \{(.*?)\};", text, flags=re.S):
        rows = re.findall(r"\{(\d+)ull, (\d+)ull\}", m.group(3))
        assert len(rows) == int(m.group(2)), m.group(1)
        found[m.group(1)] = [int(lo) | (int(hi) << 64) for lo, hi in rows]
    return found


def test_ryu_tables_device_copies_equal_host_copies_and_the_formula():
    """Every entry of both copies, recomputed with Python integers (tools/gen_ryu_tables.py's definitions): the device only
    prints doubles in about [1e-22, 1e38] through the JSON path, so most of its copy is read by nothing else in the suite."""
    t = _tables()
    assert sorted(t) == ["kPow5InvSplitDev", "kPow5InvSplitHost", "kPow5SplitDev", "kPow5SplitHost"]
    bits = 125
    inv = [(1 << ((5 ** i).bit_length() - 1 + bits)) // (5 ** i) + 1 for i in range(342)]
    pow5 = [(5 ** i) >> ((5 ** i).bit_length() - bits) if (5 ** i).bit_length() >= bits else (5 ** i) << (bits - (5 ** i).bit_length())
            for i in range(326)]
    for name, exp in (("kPow5InvSplit", inv), ("kPow5Split", pow5)):
        host, dev = t[name + "Host"], t[name + "Dev"]
        assert host == dev, (name, [i for i, (a, b) in enumerate(zip(host, dev)) if a != b][:10])
        assert dev == exp, (name, [i for i, (a, b) in enumerate(zip(dev, exp)) if a != b][:10])
        assert all(v.bit_length() <= 126 for v in dev)


def test_alignsim_32_lane_walk_equals_one_lane():
    """The pass on the host with each node's pairs split over 32 lanes (lane 0 .. 31 in turn, as alignsim_kernel splits them
    over a warp) writes the same bits and decides the same pairs as one lane, on every node size."""
    pool, nodes = node_sets(random.Random(2029))
    assert {len(nd) for nd in nodes} == set(NODE_SIZES)
    pairs1, m1 = run_nodes(pool, nodes, lanes=1)
    pairs32, m32 = run_nodes(pool, nodes, lanes=32)
    exp, modelled = expected_matrices(pool, nodes)
    assert pairs1 == pairs32 == modelled and modelled > 900000, (pairs1, pairs32, modelled)
    assert_matrices(m1, exp)
    diff = np.nonzero(m1.view(np.uint64) != m32.view(np.uint64))[0]
    assert len(diff) == 0, diff[:10]
    # and a lane count that is not a power of two: every pair is still written exactly once
    sub = nodes[:300]
    p1, a = run_nodes(pool, sub, lanes=1)
    p7, b = run_nodes(pool, sub, lanes=7)
    assert p1 == p7 and np.array_equal(a.view(np.uint64), b.view(np.uint64))
