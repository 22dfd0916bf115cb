"""The planted-optimum LP generator (tests/planted_lp.py) checked on the CPU: the GPU band-kernel tests rest on it."""
import numpy as np
import pytest

from oracle import highs as H
from oracle import lp_models as L
from planted_lp import AMAP_CASES, CASES, PLACEMENTS, UNREACHABLE, VARIANTS, band_placement, optimality, planted, shuffled

W_LIST = (0, 1, 2, 3, 4, 7, 8, 9, 16, 17, 31, 32, 33)


def _highs(p, k):
    """(objective, x) of LP k by HiGHS dual simplex at 1e-10 tolerances"""
    c, b, u, kc = p.t.instantiate(p.cparams[k], p.rparams[k])
    A = p.t.matrix(p.rparams[k])
    n = p.t.n
    lp = L.RawLP(c=c, c0=kc, A_eq=A.tocsr(), b_eq=b, A_ub=np.zeros((0, n)), b_ub=np.zeros(0), lb=np.zeros(n), ub=u,
                 names=list(p.t.col_names), meta={})
    return H.solve(lp)


@pytest.mark.parametrize("w", W_LIST)
def test_planted_bandwidth_and_kkt(w):
    """finalize() reports the requested half bandwidth; (x*, y*) satisfy the KKT conditions exactly; the margins hold"""
    for kw in (dict(), dict(bounded="all"), dict(bounded="none", extra=2), dict(amap=True, N=3)):
        p = planted(m=max(2 * w + 3, 6), w=w, seed=w, N=kw.pop("N", 2), **kw)
        assert p.t.w == w
        for k in range(p.x.shape[0]):
            o = optimality(p, k)
            assert o["primal"] == 0.0 and o["bounds"] == 0.0 and o["dual"] == 0.0 and o["sign"] == 0.0, o
            assert o["n_basic"] == p.t.m                      # nondegenerate: every basic x strictly inside
            assert o["x_margin"] >= 0.1 and o["r_margin"] >= 0.1, o


def test_planted_column_kinds_and_variants():
    assert planted(m=10, w=2, bounded="none").t.nb == 0
    p = planted(m=10, w=2, bounded="all")
    assert p.t.nb == p.t.n
    for name, kw in VARIANTS.items():
        p = planted(seed=5, N=3, **kw)
        for k in range(3):
            o = optimality(p, k)
            assert o["primal"] == 0.0 and o["bounds"] == 0.0, (name, o)
            c = p.t.instantiate(p.cparams[k], p.rparams[k])[0]
            if kw.get("zero_c"):
                assert not c.any() and p.obj[k] == p.t.instantiate(p.cparams[k], p.rparams[k])[3]
            else:
                assert o["dual"] == 0.0 and o["sign"] == 0.0, (name, o)
                assert o["r_margin"] >= 0.1 * kw.get("c_scale", 1.0), (name, o)
            if kw.get("zero_b"):
                assert not p.t.instantiate(p.cparams[k], p.rparams[k])[1].any() and not p.x[k].any()
            else:
                # (a loose box widens the range the margin is measured against)
                assert o["x_margin"] >= 0.1 * min(1.0, kw.get("b_scale", 1.0)) / kw.get("u_scale", 1.0), (name, o)


@pytest.mark.parametrize("seed", range(30))
def test_planted_agrees_with_highs(seed):
    """HiGHS finds the planted optimum: objective to 1e-9 relative, x to 1e-7"""
    rng = np.random.default_rng(seed)
    w = int(rng.choice([0, 1, 2, 3, 4, 8]))
    kw = [dict(), dict(bounded="all"), dict(bounded="none"), dict(amap=True), dict(c_scale=2.0 ** 20), dict(b_scale=2.0 ** -20)][seed % 6]
    p = planted(m=int(rng.integers(w + 2, 30)), w=w, seed=seed, N=2, **kw)
    for k in range(2):
        obj, x = _highs(p, k)
        assert abs(obj - p.obj[k]) <= 1e-9 * max(1.0, abs(p.obj[k])), (obj, p.obj[k])
        assert np.abs(x - p.x[k]).max() <= 1e-7 * max(1.0, np.abs(p.x[k]).max())


def test_shuffled_is_the_same_lp():
    p = planted(m=12, w=3, seed=4, N=2, amap=True)
    s, cperm, rperm = shuffled(p.t, seed=1)
    for k in range(2):
        c, b, u, kc = p.t.instantiate(p.cparams[k], p.rparams[k])
        c2, b2, u2, kc2 = s.instantiate(p.cparams[k], p.rparams[k])
        assert np.array_equal(c[cperm], c2) and np.array_equal(b[rperm], b2) and np.array_equal(u[cperm], u2) and kc == kc2
        assert np.array_equal(p.t.matrix(p.rparams[k]).toarray()[rperm][:, cperm], s.matrix(p.rparams[k]).toarray())


def test_band_case_table_covers_every_reachable_pair():
    """the mirror of band_geometry puts every GPU case where the table says, and the table holds every (W, placement) pair not
    documented as unreachable on an H100"""
    for (W, pl), kw in CASES.items():
        p = planted(seed=0, **kw)
        assert band_placement(p.t)[0] == pl, ((W, pl), band_placement(p.t))
    for (W, pl), kw in AMAP_CASES.items():
        assert band_placement(planted(seed=0, amap=True, **kw).t)[0] == pl, (W, pl)
    pairs = {(W, pl) for W in (1, 2, 4, 8, 16, 32) for pl in PLACEMENTS}
    assert set(CASES) == pairs - UNREACHABLE
    assert {pl for _, pl in AMAP_CASES} == set(PLACEMENTS)
