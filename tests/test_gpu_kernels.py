"""GPU parity, kernel level: CUDA K1/K2 (through the C ABI) vs the columnar C oracle, bit for bit."""
import numpy as np
import pytest

from oracle import columnar as OC
from tests.helpers import EDGE_EPS, numeric_edge_vals, random_codes, random_vals

pytestmark = pytest.mark.gpu

NONE, ABSENT = OC.F64_NONE, OC.F64_ABSENT


def _torch():
    import torch
    return torch


def same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    return np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 12, 16, 17, 31, 32, 33, 63, 64])
def test_vote_matches_oracle(n):
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(100 + n)
    F = 6
    G = F * 4099  # not a multiple of the tile
    for vocab, p_agree in ((3, 0.6), (1000, 0.3), (2, 0.9)):
        codes = random_codes(rng, G, n, vocab, p_agree=p_agree)
        none_code = np.array([-1, 0, -1, 1, vocab + 5, -1], dtype=np.int32)
        for nc in (None, none_code):
            exp_win, exp_meta = OC.vote(codes, nc)
            d_nc = torch.from_numpy(nc).cuda() if nc is not None else None
            win, meta = K.vote(torch.from_numpy(codes).cuda(), d_nc)
            torch.cuda.synchronize()
            assert np.array_equal(win.cpu().numpy(), exp_win)
            assert np.array_equal(meta.cpu().numpy().view(np.uint32), exp_meta)


@pytest.mark.parametrize("n", [8, 16, 32, 64])
def test_vote_single_field_with_none_code(n):
    """One vote field whose Nones vote (none_code given, n_fields = 1): the field index arithmetic of every front-end."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(n)
    codes = random_codes(rng, 5000, n, 4, p_none=0.3)
    for nc in (np.array([2], dtype=np.int32), np.array([-1], dtype=np.int32)):
        exp_win, exp_meta = OC.vote(codes, nc)
        win, meta = K.vote(torch.from_numpy(codes).cuda(), torch.from_numpy(nc).cuda())
        assert np.array_equal(win.cpu().numpy(), exp_win) and np.array_equal(meta.cpu().numpy().view(np.uint32), exp_meta)


@pytest.mark.parametrize("n", [2, 4, 8, 16, 32, 64])
@pytest.mark.parametrize("n_fields", [1, 2, 3, 5, 7, 9, 17, 33, 1000, 59999])
def test_vote_field_maps(n, n_fields):
    """Voting Nones with a different none_code per field, from fewer fields than vote_multi_kernel's groups per thread (the
    field wraps inside a thread's unit) up to the largest count the TMA kernels' field map takes.  The group count is odd and
    ends inside a record, so the one-group launches after vote_multi_kernel run and must pick up the field where it stopped."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(1000 * n + n_fields)
    G = max(20000, 2 * n_fields + n_fields // 2) | 1
    codes = random_codes(rng, G, n, 4, p_none=0.3, p_absent=0.02)
    none_code = rng.integers(-1, 7, n_fields).astype(np.int32)
    none_code[: min(n_fields, 2)] = (5, -1)[: min(n_fields, 2)]
    exp_win, exp_meta = OC.vote(codes, none_code)
    d_codes, d_nc = torch.from_numpy(codes).cuda(), torch.from_numpy(none_code).cuda()
    win = torch.empty(G, dtype=torch.int32, device="cuda")
    meta = torch.empty(G, dtype=torch.int32, device="cuda")
    K.check(K.load().kc_vote_i32(d_codes.data_ptr(), G, n, d_nc.data_ptr(), n_fields, win.data_ptr(), meta.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream))
    bad = np.nonzero((win.cpu().numpy() != exp_win) | (meta.cpu().numpy().view(np.uint32) != exp_meta))[0]
    assert bad.size == 0, (bad.size, bad[:5], bad[:5] % n_fields)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8, 11, 16, 24, 32, 48, 64])
@pytest.mark.parametrize("style", ["ints", "near", "pow10", "floats", "lowbits"])
def test_numeric_matches_oracle(n, style):
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(7 * n + len(style))
    G = 9001
    vals = random_vals(rng, G, n, style)
    exp_val, exp_meta = OC.numeric(vals)
    val, meta = K.numeric(torch.from_numpy(vals).cuda())
    torch.cuda.synchronize()
    got_meta = meta.cpu().numpy().view(np.uint32)
    bad = np.nonzero(got_meta != exp_meta)[0]
    assert bad.size == 0, (bad[:5], vals[bad[:1]], OC.meta_fields(got_meta[bad[:1]]), OC.meta_fields(exp_meta[bad[:1]]))
    got_val = val.cpu().numpy()
    badv = np.nonzero(got_val.view(np.uint64) != exp_val.view(np.uint64))[0]
    # NaN outputs ("no value") only need to be NaN on both sides
    badv = [i for i in badv if not (np.isnan(got_val[i]) and np.isnan(exp_val[i]))]
    assert not badv, (badv[:5], vals[badv[:1]], got_val[badv[:1]], exp_val[badv[:1]])


@pytest.mark.parametrize("n", [4, 8, 16, 32])
def test_kernels_tiny_and_ragged_group_counts(n):
    """Group counts below / around one warp and one tile: partially filled warps in the queueing fast kernels and TMA
    tiles that hang over the end of the input."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(n)
    for G in (1, 2, 31, 32, 33, 127, 129, 1000):
        vals = random_vals(rng, G, n, "ints")
        vals[:, : n // 2 + 1] = vals[:, :1]  # a majority of identical cells in most groups: the fast path decides them
        vals[rng.random((G, n)) < 0.05] = NONE
        vals = np.ascontiguousarray(vals)
        exp_val, exp_meta = OC.numeric(vals)
        val, meta = K.numeric(torch.from_numpy(vals).cuda())
        assert np.array_equal(meta.cpu().numpy().view(np.uint32), exp_meta), (n, G)
        g_, e_ = val.cpu().numpy(), exp_val
        assert ((g_.view(np.uint64) == e_.view(np.uint64)) | (np.isnan(g_) & np.isnan(e_))).all(), (n, G)
        codes = random_codes(rng, G, n, 4)
        ew, em = OC.vote(codes, None)
        w, m = K.vote(torch.from_numpy(codes).cuda(), None)
        assert np.array_equal(w.cpu().numpy(), ew) and np.array_equal(m.cpu().numpy().view(np.uint32), em), (n, G)


def test_numeric_other_eps():
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(5)
    vals = random_vals(rng, 5000, 16, "near")
    for rel, ab in ((0.0, 0.0), (0.1, 1e-3), (1e-9, 0.5)):
        exp_val, exp_meta = OC.numeric(vals, rel, ab)
        val, meta = K.numeric(torch.from_numpy(vals).cuda(), rel, ab)
        assert np.array_equal(meta.cpu().numpy().view(np.uint32), exp_meta)
        g, e = val.cpu().numpy(), exp_val
        ok = (g.view(np.uint64) == e.view(np.uint64)) | (np.isnan(g) & np.isnan(e))
        assert ok.all()


@pytest.mark.parametrize("n", [8, 16, 32])
def test_numeric_fast_path_edges(n):
    """K2's majority shortcut (kc::numeric_fast) against the oracle where it has to give up or sit on a boundary:
    neighbours right at the tolerance, cells sharing v's high word, signed zeros, -inf / negative NaN / odd NaN payloads,
    absent cells, overflow of the sum, every majority size, several (rel, abs) tolerances."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(900 + n)
    vals = numeric_edge_vals(rng, 20000, n)
    d_vals = torch.from_numpy(vals).cuda()
    for rel, ab in EDGE_EPS:
        with np.errstate(all="ignore"):
            exp_val, exp_meta = OC.numeric(vals, rel, ab)
        val, meta = K.numeric(d_vals, rel, ab)
        got_meta, g_ = meta.cpu().numpy().view(np.uint32), val.cpu().numpy()
        bad = np.nonzero(got_meta != exp_meta)[0]
        assert bad.size == 0, (rel, ab, bad[:3], vals[bad[:1]], OC.meta_fields(got_meta[bad[:1]]), OC.meta_fields(exp_meta[bad[:1]]))
        ok = (g_.view(np.uint64) == exp_val.view(np.uint64)) | (np.isnan(g_) & np.isnan(exp_val))
        assert ok.all(), (rel, ab, vals[~ok][:1], g_[~ok][:3], exp_val[~ok][:3])


def test_confidence_matches_python_round():
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(11)
    metas, pvfs, exp_v, exp_n = [], [], [], []
    for present in range(0, 65):
        for support in range(0, present + 1):
            nn = int(rng.integers(max(support, 1), present + 1)) if present else 0
            for pvf in (1.0, 0.5, 2 / 3, 0.3333333333333333, 7 / 9 * (5 / 8)):
                for flags in ((1,), (1 | 2,), (8,), (0,)):
                    f = flags[0]
                    if (f & (1 | 8)) and (support == 0 or present == 0):
                        continue
                    metas.append((3 & 0x3F) | (support << 6) | (nn << 13) | (present << 20) | (f << 27))
                    pvfs.append(pvf)
                    if f & 1:
                        exp_v.append(round(pvf * (support / present), 5))
                        exp_n.append(pvf * (1 / present) * 1.0 if f & 2 else round(support / nn, 5))
                    elif f & 8:
                        exp_v.append(pvf * (nn / present))
                        exp_n.append(pvf * (nn / present))
                    else:
                        exp_v.append(pvf if present == 0 else 0.0)
                        exp_n.append(pvf if present == 0 else 0.0)
    meta = torch.tensor(np.array(metas, dtype=np.uint32).view(np.int32)).cuda()
    pvf = torch.tensor(pvfs, dtype=torch.float64).cuda()
    got_v = K.confidence(meta, False, pvf).cpu().numpy()
    got_n = K.confidence(meta, True, pvf).cpu().numpy()
    m = np.array(metas, dtype=np.uint32)
    has = ((m >> 27) & 1) == 1
    nofin = ((m >> 27) & 8) == 8
    # vote confidences are defined for HAS_VALUE / no-value words; numeric for all four kinds
    sel_v = has | (~has & ~nofin)
    assert np.array_equal(got_v[sel_v], np.array(exp_v)[sel_v])
    assert np.array_equal(got_n, np.array(exp_n))


def test_round5_random_products():
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(3)
    # confidence = round(pvf * support/present, 5) for arbitrary pvf in (0, 1]
    present = rng.integers(1, 65, 200000)
    support = (rng.random(200000) * present).astype(np.int64) + 1
    support = np.minimum(support, present)
    pvf = rng.random(200000)
    pvf[:1000] = np.round(pvf[:1000], 5) + 5e-6  # near-half cases
    meta = ((support << 6) | (present << 13) | (present << 20) | (1 << 27)).astype(np.uint32)
    got = K.confidence(torch.tensor(meta.view(np.int32)).cuda(), False, torch.tensor(pvf).cuda()).cpu().numpy()
    exp = np.array([round(float(p) * (int(s) / int(t)), 5) for p, s, t in zip(pvf, support, present)])
    assert np.array_equal(got, exp)


def test_logprob_sum_matches_oracle():
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(17)
    lens = rng.integers(0, 200, 5000)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    lp = (-rng.exponential(1.0, offsets[-1])).astype(np.float32)
    exp = OC.logprob_sum(lp, offsets)
    got = K.logprob_sum(torch.from_numpy(lp).cuda(), torch.from_numpy(offsets).cuda()).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))
    ref64 = np.array([lp[offsets[i]:offsets[i + 1]].astype(np.float64).sum() for i in range(len(lens))])
    assert np.max(np.abs(got - ref64)) < 1e-3  # fp32 accumulation error at |sum| ~ 200; the spec is the fixed order above


def test_s32_full_size_properties():
    """BASELINE config 2 at full size (1M x 32 fields, n=16): size-independent properties."""
    torch = _torch()
    from k_llms_b200 import _native as K
    from k_llms_b200 import synth
    N, n = 1_000_000, 16
    codes, none_code, vals = synth.s32_torch(N, n, 20260923, "cuda")
    win, meta = K.vote(codes.view(N * 24, n), none_code)
    value, nmeta = K.numeric(vals.view(N * 8, n))
    torch.cuda.synchronize()
    m = meta.view(N, 24).to(torch.int64) & 0xFFFFFFFF
    idx, support, nn, present = m & 0x3F, (m >> 6) & 0x7F, (m >> 13) & 0x7F, (m >> 20) & 0x7F
    has = ((m >> 27) & 1) == 1
    c3 = codes.to(torch.int64)
    eff = torch.where(c3 == -1, none_code.view(1, 24, 1).to(torch.int64), c3)
    assert bool((present == n).all())
    assert bool((nn == (eff >= 0).sum(-1)).all())
    # the winner's count is what the result word says, and no class beats it
    w = win.view(N, 24, 1).to(torch.int64)
    assert bool((((eff == w) & (eff >= 0)).sum(-1) == support)[has].all())
    onehot_max = torch.zeros_like(support)
    for code in range(8):
        onehot_max = torch.maximum(onehot_max, (eff == code).sum(-1))
    assert bool((onehot_max == support).all())
    # first-seen: cell idx holds the winner, and no earlier cell does
    first = torch.gather(eff, 2, idx.unsqueeze(-1)).squeeze(-1)
    assert bool((first == win.view(N, 24))[has].all())
    pos = torch.arange(n, device="cuda").view(1, 1, n)
    earlier = ((eff == w) & (pos < idx.unsqueeze(-1))).any(-1)
    assert not bool(earlier[has].any())
    # idempotence: consensus of n copies of the consensus is the consensus
    again, meta2 = K.vote(win.view(-1, 1).expand(-1, n).contiguous(), None)
    assert bool((again == win).all())
    # numeric: a value exists wherever >= 1 finite cell; it lies inside [min, max] of the finite cells
    v = vals
    fin = torch.isfinite(v)
    lo = torch.where(fin, v, torch.full_like(v, float("inf"))).amin(-1)
    hi = torch.where(fin, v, torch.full_like(v, float("-inf"))).amax(-1)
    val = value.view(N, 8)
    ok = (val >= lo * (1 - 1e-15)) & (val <= hi * (1 + 1e-15))  # np.mean of k equal floats may round by an ulp
    assert bool(ok[fin.any(-1)].all())
    # sample 20k records against the C oracle bit for bit
    sel = torch.randperm(N, device="cuda")[:20000]
    ew, em = OC.vote(codes[sel].cpu().numpy().reshape(-1, n), none_code.cpu().numpy())
    assert np.array_equal(win.view(N, 24)[sel].cpu().numpy().reshape(-1), ew)
    assert np.array_equal(meta.view(N, 24)[sel].cpu().numpy().reshape(-1).view(np.uint32), em)
    ev, enm = OC.numeric(vals[sel].cpu().numpy().reshape(-1, n))
    assert np.array_equal(value.view(N, 8)[sel].cpu().numpy().reshape(-1).view(np.uint64), ev.view(np.uint64))
    assert np.array_equal(nmeta.view(N, 8)[sel].cpu().numpy().reshape(-1).view(np.uint32), enm)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 8, 12, 16, 24, 32, 48, 64])
def test_weighted_vote_matches_oracle(n):
    """K3b (self-defined spec, DESIGN.md §5): bit-exact against the C oracle, incl. the class weights."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(40 + n)
    R, F = 3001, 5
    codes = random_codes(rng, R * F, n, 4, p_agree=0.5).reshape(R, F, n)
    lp = (-rng.exponential(6.0, (R, n))).astype(np.float32)
    lp[rng.random((R, n)) < 0.02] = -500.0  # hopeless candidates (weight underflows to the clamp)
    none_code = np.array([-1, 0, -1, 2, -1], dtype=np.int32)
    for nc in (None, none_code):
        ew, em, ewt = OC.weighted_vote(codes, lp, nc)
        win, meta, wt = K.weighted_vote(torch.from_numpy(codes).cuda(), torch.from_numpy(lp).cuda(),
                                        torch.from_numpy(nc).cuda() if nc is not None else None)
        assert np.array_equal(win.cpu().numpy(), ew)
        assert np.array_equal(meta.cpu().numpy().view(np.uint32), em)
        assert np.array_equal(wt.cpu().numpy().view(np.uint32), ewt.view(np.uint32))


def test_config4_logprob_pipeline_n32():
    """BASELINE config 4 shape (n=32, ragged per-token logprobs): K3 sums -> K3b weighted vote, against the oracle,
    plus the fp64 deviation of the fp32 likelihood sums (reported, since fp32 cannot hold 1e-6 at |sum| ~ 40)."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(4)
    R, F, n = 4096, 8, 32
    lens = rng.integers(8, 65, R * n)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    lp = (-rng.exponential(1.0, offsets[-1])).astype(np.float32)
    codes = random_codes(rng, R * F, n, 6, p_absent=0.0).reshape(R, F, n)
    sums = K.logprob_sum(torch.from_numpy(lp).cuda(), torch.from_numpy(offsets).cuda())
    exp_sums = OC.logprob_sum(lp, offsets)
    assert np.array_equal(sums.cpu().numpy().view(np.uint32), exp_sums.view(np.uint32))
    win, meta, wt = K.weighted_vote(torch.from_numpy(codes).cuda(), sums.view(R, n))
    ew, em, ewt = OC.weighted_vote(codes, exp_sums.reshape(R, n))
    assert np.array_equal(win.cpu().numpy(), ew) and np.array_equal(meta.cpu().numpy().view(np.uint32), em)
    assert np.array_equal(wt.cpu().numpy().view(np.uint32), ewt.view(np.uint32))
    ref64 = np.add.reduceat(lp.astype(np.float64), offsets[:-1])
    assert np.max(np.abs(exp_sums - ref64)) < 1e-4


def test_config4_full_size_256k_n32():
    """BASELINE config 4 AT SIZE: 262,144 records x 24 vote fields, n = 32, ragged per-token logprobs (8..64 tokens): K3 then
    K3b on the device; a 3,000-record sample against the C oracle bit for bit, and size-independent properties on everything:
    the winner is one of the group's voting codes, its weight share lies in (0, 1], the winning class holds the group's heaviest
    voter or outweighs it, and a second run gives identical bits (self-defined semantics, DESIGN.md section 5)."""
    torch = _torch()
    from k_llms_b200 import _native as K
    R, F, n = 262_144, 24, 32
    g = torch.Generator(device="cuda").manual_seed(20260921 + 4)
    lens = torch.randint(8, 65, (R * n,), generator=g, device="cuda", dtype=torch.int64)
    offsets = torch.zeros(R * n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offsets[1:])
    lp = -torch.empty(int(offsets[-1].item()), dtype=torch.float32, device="cuda").exponential_(1.0, generator=g)
    truth = torch.randint(0, 6, (R, F, 1), generator=g, device="cuda", dtype=torch.int32)
    noise = torch.randint(0, 6, (R, F, n), generator=g, device="cuda", dtype=torch.int32)
    codes = torch.where(torch.rand((R, F, n), generator=g, device="cuda") < 0.8, truth.expand(-1, -1, n), noise)
    codes = torch.where(torch.rand((R, F, n), generator=g, device="cuda") < 0.05, torch.full_like(codes, -1), codes).contiguous()
    sums = K.logprob_sum(lp, offsets)
    win, meta, wt = K.weighted_vote(codes, sums.view(R, n))
    win2, meta2, wt2 = K.weighted_vote(codes, sums.view(R, n))
    assert torch.equal(win, win2) and torch.equal(meta, meta2) and torch.equal(wt.view(torch.int32), wt2.view(torch.int32))
    # sample against the oracle
    S = 3000
    o_h, lp_h = offsets[:S * n + 1].cpu().numpy(), lp[:int(offsets[S * n].item())].cpu().numpy()
    e_sums = OC.logprob_sum(lp_h, o_h)
    assert np.array_equal(sums[:S * n].cpu().numpy().view(np.uint32), e_sums.view(np.uint32))
    ew, em, ewt = OC.weighted_vote(codes[:S].cpu().numpy(), e_sums.reshape(S, n))
    assert np.array_equal(win[:S * F].cpu().numpy(), ew) and np.array_equal(meta[:S * F].cpu().numpy().view(np.uint32), em)
    assert np.array_equal(wt[:S * F].cpu().numpy().view(np.uint32), ewt.view(np.uint32))
    # properties over all 6.3 M groups
    c2 = codes.view(R * F, n)
    has = (c2 >= 0).any(dim=1)
    assert torch.equal(has, ((meta >> 27) & 1).bool())
    member = (c2 == win.view(-1, 1)).any(dim=1)
    assert bool((member | ~has).all())
    assert bool(((wt > 0) & (wt <= 1.0))[has].all()) and bool((wt[~has] == 0).all())
    w_seq = sums.view(R, 1, n).expand(R, F, n).reshape(R * F, n)
    heavy = torch.where(c2 >= 0, w_seq, torch.full_like(w_seq, -3.0e38)).argmax(dim=1, keepdim=True)
    heavy_code = torch.gather(c2, 1, heavy).view(-1)
    assert bool(((wt >= 0.5) | (heavy_code != win) | ~has | (wt > 0)).all())
    share_of_heavy_class = (heavy_code == win)[has].float().mean().item()
    assert share_of_heavy_class > 0.9  # the class of the heaviest voter almost always wins: the walk's first pick


def test_logprob_sum_staged_tiles_and_fallback():
    """K3's shared-memory-staged kernel (>= 4096 sequences): empty and 1-token sequences, lengths around the 32-lane
    stride, tiles whose tokens exceed the staging buffer (warp-per-sequence fallback inside the kernel), -0.0 inputs."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(12)
    S = 20000
    lens = rng.choice([0, 1, 2, 31, 32, 33, 63, 64, 65, 95, 96, 97, 200], S)
    lens[5000:5003] = [30000, 7, 15000]        # tiles 39: far beyond the buffer
    lens[12800:12928] = 97                     # a full tile just above 12288 tokens
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    lp = (-rng.exponential(1.0, offsets[-1])).astype(np.float32)
    lp[rng.random(lp.size) < 0.01] = -0.0
    got = K.logprob_sum(torch.from_numpy(lp).cuda(), torch.from_numpy(offsets).cuda()).cpu().numpy()
    exp = OC.logprob_sum(lp, offsets)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


@pytest.mark.parametrize("n", [8, 16, 32, 64])
@pytest.mark.parametrize("fields", [1, 4, 5, 24, 200])
def test_weighted_vote_per_record_kernel(n, fields):
    """K3b's weights-once-per-record kernel over several fields-per-record shapes (tiles spanning 1 .. 128 records)."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(n * 1000 + fields)
    R = max(2, 30000 // fields)
    codes = random_codes(rng, R * fields, n, 5, p_absent=0.05).reshape(R, fields, n)
    none_code = rng.choice([-1, 0, 3], fields).astype(np.int32)
    # skewed weights; then weights from a two-value set (equal class weights are common: ties, first-seen rule, and the
    # heaviest candidate is rarely in the first-seen class)
    for seq in ((-rng.exponential(20.0, (R, n))).astype(np.float32), rng.choice([-1.0, -1.0, -2.0], (R, n)).astype(np.float32),
                np.zeros((R, n), dtype=np.float32)):
        for nc in (None, none_code):
            win, meta, wt = K.weighted_vote(torch.from_numpy(codes).cuda(), torch.from_numpy(seq).cuda(),
                                            torch.from_numpy(nc).cuda() if nc is not None else None)
            ew, em, ewt = OC.weighted_vote(codes, seq, nc)
            assert np.array_equal(win.cpu().numpy(), ew) and np.array_equal(meta.cpu().numpy().view(np.uint32), em)
            assert np.array_equal(wt.cpu().numpy().view(np.uint32), ewt.view(np.uint32))


@pytest.mark.parametrize("n", [32, 64])
def test_weighted_vote_many_fields_per_record_fallback(n):
    """At n = 32 and 64, 60000 fields or more per record leave the TMA kernels (their field map stops below 60000) for the
    per-record kernel."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(60000 + n)
    R, F = 3, 60000
    codes = random_codes(rng, R * F, n, 5, p_none=0.2, p_absent=0.05).reshape(R, F, n)
    seq = (-rng.exponential(4.0, (R, n))).astype(np.float32)
    none_code = rng.integers(-1, 6, F).astype(np.int32)
    for nc in (None, none_code):
        win, meta, wt = K.weighted_vote(torch.from_numpy(codes).cuda(), torch.from_numpy(seq).cuda(),
                                        torch.from_numpy(nc).cuda() if nc is not None else None)
        ew, em, ewt = OC.weighted_vote(codes, seq, nc)
        assert np.array_equal(win.cpu().numpy(), ew) and np.array_equal(meta.cpu().numpy().view(np.uint32), em)
        assert np.array_equal(wt.cpu().numpy().view(np.uint32), ewt.view(np.uint32))

@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8, 16, 17, 32, 33, 64])
def test_vote_i8_equals_i32(n):
    """Compact int8 cells are a lossless input format: same outputs as the int32 path and as the oracle."""
    torch = _torch()
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(900 + n)
    F = 5
    codes = random_codes(rng, F * 2003, n, 7)
    none_code = np.array([-1, 0, 3, -1, -1], dtype=np.int32)
    for nc in (None, none_code):
        ew, em = OC.vote(codes, nc)
        d_nc = torch.from_numpy(nc).cuda() if nc is not None else None
        win, meta = K.vote_i8(torch.from_numpy(codes.astype(np.int8)).cuda(), d_nc)
        assert np.array_equal(win.cpu().numpy(), ew)
        assert np.array_equal(meta.cpu().numpy().view(np.uint32), em)


def test_host_entry_int8_cells():
    from k_llms_b200 import _native as K
    from k_llms_b200 import synth
    codes, none_code, vals = synth.s32_numpy(50_003, 16, 9)
    a = K.consensus_host(codes, none_code, vals)
    b = K.consensus_host(codes.astype(np.int8), none_code, vals)
    for k in ("win_code", "vote_meta", "num_meta"):
        assert np.array_equal(a[k], b[k])
    assert np.array_equal(a["value"].view(np.uint64), b["value"].view(np.uint64))


def test_medoid_kernel_matches_oracle():
    """K4 == ko_medoid_str (pinned to the reference in tests/golden/medoid.json) on random phrase groups: index and mean bit-exact."""
    from k_llms_b200 import _native
    from k_llms_b200.columnar import _normalize
    from tests.helpers import random_string_groups
    torch = _torch()
    rng = np.random.default_rng(77)
    groups = [[_normalize(s) for s in g] for g in random_string_groups(rng, 3000, max_k=64)]
    groups += [["a", "a"], ["", ""], ["", "abc", ""], ["x" * 64, "y" * 64, "x" * 63 + "y"], ["abc"] * 64,
               ["a" * 32, "a" * 31 + "b", "b" * 33, "a" * 32], ["q" * 64, "q" * 500 + "z", "q" * 10, "zq" * 16],
               ["ab" * 16 + "c", "ab" * 16, "ba" * 16, "ab" * 16 + "c", "ab" * 17]]
    chars, str_off, grp_off = OC.pack_string_groups(groups)
    exp_idx, exp_avg = OC.medoid(groups)
    idx, avg = _native.medoid_str(torch.from_numpy(chars).cuda(), torch.from_numpy(str_off).cuda(), torch.from_numpy(grp_off).cuda(),
                                  max_group=max(len(g) for g in groups))
    torch.cuda.synchronize()
    assert np.array_equal(idx.cpu().numpy(), exp_idx)
    assert same_bits(avg.cpu().numpy(), exp_avg)
    small = [g[:5] for g in groups]  # another shared-memory geometry (max_group = 5)
    chars, str_off, grp_off = OC.pack_string_groups(small)
    exp_idx, exp_avg = OC.medoid(small)
    idx, avg = _native.medoid_str(torch.from_numpy(chars).cuda(), torch.from_numpy(str_off).cuda(), torch.from_numpy(grp_off).cuda(),
                                  max_group=5)
    assert np.array_equal(idx.cpu().numpy(), exp_idx) and same_bits(avg.cpu().numpy(), exp_avg)
