"""K2's majority shortcut with one or two cells chained to the majority value (kc::numeric_fast_decide's walk and
numeric_fast_finish's sum with extras) against the columnar C oracle, bit for bit, at the three fast-kernel sizes."""
import numpy as np
import pytest

from oracle import columnar as OC
from tests.helpers import EDGE_EPS, _down, _up

pytestmark = pytest.mark.gpu

NONE, ABSENT = OC.F64_NONE, OC.F64_ABSENT


def _extras(rng, v, rel, ab):
    """One to three values around v that hit a branch of the walk: inside / on / one ulp past the tolerance, chained to
    a third cell just inside or outside reach, sharing v's or each other's high word, negative, signed zeros."""
    reach = max(ab, rel * max(abs(v), 1.0))
    e_in_lo, e_in_hi = v - reach * 0.5, v + reach * 0.5
    edge_lo, edge_hi = v - reach, v + reach
    kind = int(rng.integers(0, 12))
    if kind == 0:
        return [e_in_lo]
    if kind == 1:
        return [e_in_hi]
    if kind == 2:
        return [e_in_lo, v - reach * 0.9]
    if kind == 3:
        return [e_in_hi, v + reach * 0.9]
    if kind == 4:
        return [e_in_lo, e_in_hi]
    if kind == 5:  # at the edge and one or two ulps beyond
        return [float(rng.choice([edge_lo, _down(edge_lo), _up(edge_lo), edge_hi, _up(edge_hi), _down(edge_hi, 2)]))]
    if kind == 6:  # a chain: the third cell just inside or just outside the reach of the second
        e = e_in_hi
        r2 = max(ab, rel * max(abs(e), 1.0))
        return [e, float(rng.choice([e + r2 * 0.999, _up(e + r2), e + r2 * 1.001]))]
    if kind == 7:  # three extras in a chain
        return [e_in_lo, v - reach, v - reach * 1.4]
    if kind == 8:  # sharing v's high word, or each other's
        return [float(rng.choice([_up(v), _down(v, 3)]))] if rng.random() < 0.5 else [e_in_hi, _up(e_in_hi)]
    if kind == 9:
        return [-e_in_hi if v != 0 else -5e-324]
    if kind == 10:
        return [0.0, -0.0][: int(rng.integers(1, 3))]
    return [e_in_lo, v * 3.0 + 1.0]  # an extra and a far cell


def neighbour_vals(rng, G, n, rel, ab):
    pool = np.array([1000.0, 123456.0, 1.0, 0.1, 0.0, 5e-324, 3.3, 1e15 + 0.5, 2.0 ** 52, 999999.0, 1.7e308], dtype=np.float64)
    rows = np.empty((G, n), dtype=np.float64)
    for g in range(G):
        v = float(pool[rng.integers(0, len(pool))])
        with np.errstate(all="ignore"):
            ex = [x for x in _extras(rng, v, rel, ab) if np.isfinite(x)]
        c = int(rng.integers(n // 2 + 1, n + 1))  # every residue of c mod 8 over the draws
        row = [v] * c + ex[: n - c]
        while len(row) < n:  # None / absent cells and far values
            row.append(float(rng.choice([NONE, ABSENT, NONE, v * 5.0 + 7.0])))
        rows[g] = rng.permutation(np.array(row, dtype=np.float64))
    return rows


@pytest.mark.parametrize("n", [8, 16, 32])
def test_numeric_neighbours_match_oracle(n):
    import torch
    from k_llms_b200 import _native as K
    rng = np.random.default_rng(4200 + n)
    for rel, ab in EDGE_EPS:
        for G in (1, 31, 33, 20000 + 17):  # group counts that end inside a tile
            vals = neighbour_vals(rng, G, n, rel, ab)
            with np.errstate(all="ignore"):
                exp_val, exp_meta = OC.numeric(vals, rel, ab)
            val, meta = K.numeric(torch.from_numpy(vals).cuda(), rel, ab)
            got_meta, got = meta.cpu().numpy().view(np.uint32), val.cpu().numpy()
            bad = np.nonzero(got_meta != exp_meta)[0]
            assert bad.size == 0, (n, rel, ab, G, vals[bad[:1]], OC.meta_fields(got_meta[bad[:1]]), OC.meta_fields(exp_meta[bad[:1]]))
            ok = (got.view(np.uint64) == exp_val.view(np.uint64)) | (np.isnan(got) & np.isnan(exp_val))
            assert ok.all(), (n, rel, ab, G, vals[~ok][:1], got[~ok][:3], exp_val[~ok][:3])
