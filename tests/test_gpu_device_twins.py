"""GPU: the device instantiations of code that is written once as __host__ __device__ and checked strictly on the host,
held to the same exact references on the device.

- The number conversions of the device JSON path (kc_jsoncore.cuh: to_double, float_repr) run on the GPU against CPython's
  float() and repr, and against their host instantiation's accept / decline flags; then every number through the device
  JSON path, one record per number.
- The structured JSON fuzz and the mutated records through both device JSON entry points (count and likelihood-weighted
  votes): the same records accepted as by the host instantiation of the phases, byte-identical texts, the same bytes on
  every run and under any chunking.
- The element-similarity pass of the alignment (kc_alignsim.cuh) with its 32-lane pair walk, bit for bit against the host.
- K4 under the jaccard / hamming methods (kc_medoid.cuh) against a plain restatement, including its exact duplicate scan
  (groups of more than 32 strings, and a 32-bit FNV-1a collision)."""
import json
import random

import numpy as np
import pytest

from k_llms_b200 import _native as K
from tests.alignsim_cases import NODE_SIZES, assert_matrices, expected_matrices, node_sets, run_nodes
from tests.helpers import (_fnv1a, _fnv_collision, boundary_texts, general_and_mutated_records, jsongpu_with_oracle, near_halfway_texts,
                           number_texts, repr_doubles)
from tests.test_gpu_json import _expected
from tests.test_json_fuzz import _records
from tests.test_jsongpu_host_logic import assert_parsed_like_cpython, parse_doubles
from tests.test_weighted_host_logic import _seq

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


# ----------------------------------------------------------------------------- A. number conversions

def _number_corpus():
    """(texts, index of the first text that must be declined, count of near-halfway texts)."""
    near = near_halfway_texts()
    edges, decline = boundary_texts()
    texts = number_texts() + near + edges
    return texts + decline, len(texts), len(near)


def _reprs(xs, device=None):
    lib = K.load()
    buf, lens = np.zeros((len(xs), 32), dtype=np.uint8), np.zeros(len(xs), dtype=np.int32)
    if device is None:
        K.check(lib.kc_debug_float_reprs(xs.ctypes.data, len(xs), buf.ctypes.data, lens.ctypes.data))
    else:
        K.check(lib.kc_debug_float_reprs_device(xs.ctypes.data, len(xs), buf.ctypes.data, lens.ctypes.data, device))
    return buf, lens


def test_number_conversions_on_the_device():
    """to_double and float_repr run by one GPU thread per value: float(text) bit for bit, json.dumps(x) byte for byte, and the
    same accept / decline flag as the host instantiation on every text."""
    _torch()
    texts, first_decline, n_near = _number_corpus()
    out, ok = parse_doubles(texts, device=0)
    h_out, h_ok = parse_doubles(texts)
    assert np.array_equal(ok, h_ok), [texts[i] for i in np.nonzero(ok != h_ok)[0][:10]]
    assert not ok[first_decline:].any()
    assert ok.sum() > 0.8 * len(texts)
    assert_parsed_like_cpython(texts, out, ok)
    assert np.array_equal(out[ok == 1].view(np.uint64), h_out[ok == 1].view(np.uint64))

    xs = np.ascontiguousarray(np.concatenate([repr_doubles(), out[ok == 1], -out[ok == 1]]))
    buf, lens = _reprs(xs, device=0)
    h_buf, h_lens = _reprs(xs)
    assert np.array_equal(lens, h_lens) and np.array_equal(buf, h_buf)
    bad = [i for i, x in enumerate(xs.tolist()) if bytes(buf[i, :lens[i]]) != json.dumps(x).encode()]
    assert not bad, [(xs[i], bytes(buf[i, :lens[i]])) for i in bad[:10]]
    print(f"\nnumber conversions on the device: {len(texts)} texts ({n_near} near-halfway, {int(ok.sum())} accepted), "
          f"{len(xs)} doubles printed")


def _run_packed(records, flags=K.JSON_DEVICE_ONLY, seq=None):
    blob, off, n = K.pack_texts(records)
    if seq is None:
        res = K.consolidate_json_packed(blob, off, n, flags=flags)
    else:
        res = K.consolidate_json_packed_weighted(blob, off, n, seq, flags=flags)
    try:
        return res.pairs(), np.array(res.status), np.array(res.why), res.stats.chunks
    finally:
        res.close()


def test_numbers_through_the_device_json_path():
    """One number per record, so that a declined number hides nothing else: {"x": t} twice (K2's pair mean, exact here) and
    {"x": t} with {"x": null} (the cell comes back unchanged).  Acceptance equals the host instantiation's; accepted
    contents equal CPython's, likelihoods the oracle's."""
    _torch()
    texts, _, _ = _number_corpus()
    values = [json.loads(t) for t in texts]
    rng = random.Random(3)
    for kind in ("pair", "null"):
        records = [['{"x": %s}' % t, '{"x": %s}' % (t if kind == "pair" else "null")] for t in texts]
        got, status, why = _run_packed(records)[:3]
        host, _ = jsongpu_with_oracle(records)
        assert [p is None for p in got] == [p is None for p in host]
        assert (why[status != 0] != 0).all()
        accepted = 0
        for r, (g, h, v) in enumerate(zip(got, host, values)):
            if g is None:
                continue
            accepted += 1
            # the pair mean is Python's sum of the two (from 0: -0.0 comes out 0.0) over two; a lone cell prints as parsed
            content = json.dumps(sum([float(v), float(v)]) / 2) if kind == "pair" else json.dumps(v)
            assert g == h and g[0] == '{"x": %s}' % content, (texts[r], g, h)
        for r in rng.sample([r for r, g in enumerate(got) if g is not None], 3000):
            assert got[r] == _expected(records[r]), (records[r], got[r])
        assert accepted > 0.8 * len(records), (kind, accepted)
        print(f"\nnumbers through the device JSON path ({kind}): {accepted} of {len(records)} records accepted")


# ----------------------------------------------------------------------------- B. the JSON fuzz on the device

def _fuzz_batches():
    """(label, records): the structured fuzz at n in {2, 3, 5, 8, 16} as generated and at n = 33 and 64, then the general and
    mutated records of the device JSON path's tests."""
    for n, recs in sorted(_records(8000, 424242).items()):
        yield f"fuzz n={n}", recs
    yield "fuzz n=33", _records(160, 33, ns=(33,))[33]
    yield "fuzz n=64", _records(100, 64, ns=(64,))[64]
    for n, recs in sorted(general_and_mutated_records(11).items()):
        yield f"mutated n={n}", recs


def _replicated(records, min_bytes=3 << 20):
    size = sum(len(t) for r in records for t in r)
    return records * (min_bytes // max(size, 1) + 1)


@pytest.mark.parametrize("weighted", [False, True], ids=["count", "weighted"])
def test_json_fuzz_on_the_device(monkeypatch, weighted):
    """Every record the device accepts equals its host instantiation (and, for count votes, the reference's client order)
    byte for byte, and the device declines exactly the records the host instantiation declines.  Run twice and once more
    in 1 MB chunks, the outputs are the same bytes: the order in which the slots phase claims rows must not show."""
    _torch()
    rng = np.random.default_rng(5 + weighted)
    total = 0
    for label, recs in _fuzz_batches():
        n = len(recs[0])
        seq = np.concatenate([_seq(rng, n) for _ in recs]).astype(np.float32) if weighted else None
        got, status, why, _ = _run_packed(recs, seq=seq)
        host, host_status = jsongpu_with_oracle(recs, seq) if weighted else jsongpu_with_oracle(recs)
        assert [p is None for p in got] == [s != 0 for s in host_status], label
        assert (why[status != 0] != 0).all(), label
        accepted = 0
        for texts, g, h in zip(recs, got, host):
            if g is None:
                continue
            accepted += 1
            assert g == h, (label, texts, g, h)
            if not weighted:
                assert g == _expected(texts), (label, texts, g)
        total += accepted
        print(f"\n{'weighted' if weighted else 'count'} votes, {label}: {accepted} of {len(recs)} records accepted on the device")
        big = _replicated(recs)
        big_seq = np.tile(seq, len(big) // len(recs)) if weighted else None
        first = _run_packed(big, seq=big_seq)
        assert first[0][:len(recs)] == got, label
        again = _run_packed(big, seq=big_seq)
        monkeypatch.setenv("KC_JSON_CHUNK_MB", "1")
        chunked = _run_packed(big, seq=big_seq)
        monkeypatch.delenv("KC_JSON_CHUNK_MB")
        assert chunked[3] > 1, (label, chunked[3])
        for other in (again, chunked):
            assert other[0] == first[0] and np.array_equal(other[1], first[1]), label
    print(f"\n{'weighted' if weighted else 'count'} votes: {total} fuzz and mutated records accepted on the device")
    assert total > 2500, total


# ----------------------------------------------------------------------------- C. alignment similarity matrices

def test_alignsim_matrices_on_the_device():
    """alignsim_kernel over thousands of list nodes of every size (warps, CTAs and the grid stride each take several):
    every cell equals the host phase's bits, every modelled pair equals generic_similarity, NaN elsewhere and on the
    diagonal, and the decided-pair count equals the host's."""
    _torch()
    pool, nodes = node_sets(random.Random(2029))
    assert {len(nd) for nd in nodes} == set(NODE_SIZES)
    pairs, got = run_nodes(pool, nodes, device=0)
    h_pairs, host = run_nodes(pool, nodes, lanes=1, device=-1)
    assert pairs == h_pairs, (pairs, h_pairs)
    diff = np.nonzero(got.view(np.uint64) != host.view(np.uint64))[0]
    assert len(diff) == 0, (len(diff), diff[:10])
    exp, modelled = expected_matrices(pool, nodes)
    assert_matrices(got, exp)
    assert modelled == pairs
    print(f"\nalignment similarities: {len(nodes)} nodes, {pairs} pairs decided on the device")


# ----------------------------------------------------------------------------- D. K4 under jaccard / hamming

def _sim(a, b, method):
    if a == b:
        return 1.0
    if method == "jaccard":
        A, B = set(a), set(b)
        return max(1e-8, len(A & B) / len(A | B)) if A | B else 1.0
    m = max(len(a), len(b))
    d = sum(x != y for x, y in zip(a, b)) + abs(len(a) - len(b))  # the shorter padded with blanks: a pad never matches
    return max(1e-8, 1 - d / m)


def _medoid(group, method):
    k = len(group)
    M = np.full((k, k), np.nan)
    for i in range(k):
        for j in range(k):
            if i != j:
                M[i, j] = _sim(group[i], group[j], method)
    means = np.nanmean(M, axis=1)
    i = int(np.argmax(means))
    return i, float(means[i])


_LENGTHS = (0, 1, 2, 5, 9, 17, 31, 32, 33, 63, 64, 65, 199, 200, 203)


def _k4_groups(rng, n_groups, max_group, collision):
    groups = []
    for g in range(n_groups):
        k = int(rng.integers(2, max_group + 1))
        if max_group == 64 and g % 5 < 3:
            k = (32, 33, 64)[g % 5]
        letters = rng.choice(list("abcdefghijklmnopqrstuvwxyz0123456789"), int(rng.integers(2, 37)), replace=False)
        base = "".join(rng.choice(letters, int(rng.choice(_LENGTHS))))
        grp = []
        for _ in range(k):
            r = rng.random()
            if grp and r < 0.25:                      # a duplicate of an earlier member
                s = grp[int(rng.integers(0, len(grp)))]
            elif r < 0.6 and base:                    # the base with a few substitutions, a cut or an extension
                s = list(base)
                for _ in range(int(rng.integers(0, 4))):
                    s[int(rng.integers(0, len(s)))] = str(rng.choice(letters))
                s = "".join(s)[: int(rng.integers(0, len(s) + 1))] if rng.random() < 0.2 else "".join(s)
                s = s + "".join(rng.choice(letters, int(rng.integers(0, 3))))
            elif r < 0.67:
                s = ""                                # normalised to nothing
            else:
                s = "".join(rng.choice(letters, int(rng.choice(_LENGTHS))))
            grp.append(s)
        if g % 7 == 0 and k <= 32:                    # the hash-colliding pair: the exact scan in a group of <= 32
            i, j = rng.choice(k, 2, replace=False)
            grp[int(i)], grp[int(j)] = collision
        groups.append(grp)
    return groups


@pytest.mark.parametrize("method", ["jaccard", "hamming"])
def test_k4_jaccard_hamming_against_a_restatement(method):
    """kc_medoid_str_method under `method` at three max_group geometries: the medoid index and its mean similarity equal
    the restatement's (set / padded-mismatch formula floored at 1e-8, np.nanmean with a NaN diagonal, np.argmax)."""
    torch = _torch()
    a, b = _fnv_collision()
    h = _fnv1a(np.frombuffer((a + b).encode(), np.uint8).reshape(2, 8))
    assert a != b and h[0] == h[1]
    rng = np.random.default_rng(61 if method == "jaccard" else 62)
    over32 = with_collision = 0
    for max_group, n_groups in ((5, 300), (20, 300), (64, 240)):
        groups = _k4_groups(rng, n_groups, max_group, (a, b))
        flat = [s for g in groups for s in g]
        chars = np.frombuffer("".join(flat).encode() or b"\0", dtype=np.uint8)
        str_off = np.concatenate([[0], np.cumsum([len(s) for s in flat])]).astype(np.int32)
        grp_off = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int32)
        idx, avg = K.medoid_str(torch.from_numpy(chars.copy()).cuda(), torch.from_numpy(str_off).cuda(), torch.from_numpy(grp_off).cuda(),
                                max_group=max_group, method=method)
        idx, avg = idx.cpu().numpy(), avg.cpu().numpy()
        for g, grp in enumerate(groups):
            ei, ea = _medoid(grp, method)
            assert (int(idx[g]), np.float64(avg[g]).tobytes()) == (ei, np.float64(ea).tobytes()), (max_group, grp, idx[g], avg[g], ei, ea)
            over32 += len(grp) > 32
            with_collision += a in grp and b in grp and len(grp) <= 32
    assert over32 > 100 and with_collision > 20, (over32, with_collision)
    print(f"\nK4 {method}: {over32} groups with k > 32, {with_collision} groups of <= 32 holding an FNV-1a collision")
