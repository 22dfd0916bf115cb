"""CPU tests of the sensitivity post-pass (dsp_lp_sensitivities): its source on the SIMT emulator against the numpy mirror, and the
mirror's definition against exact optima of real, degenerate dispatch LPs."""
import shutil
import sys
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import scenarios as SC, templates as TP  # noqa: E402
import exact_lp as E  # noqa: E402
import real_lps as R  # noqa: E402
import sensitivity_numpy as SN  # noqa: E402

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")
EMU_REL = 1e-13


def _inputs(t, N, seed, amap_rp=None):
    """random (cparams, rparams, x, y) of the template's shapes: the pass is a fixed linear map of them, optimal or not"""
    rng = np.random.default_rng(seed)
    cp = rng.normal(30.0, 20.0, (N, t.Pc))
    rp = np.abs(rng.normal(50.0, 30.0, (N, t.Pr))) if amap_rp is None else np.broadcast_to(amap_rp, (N, t.Pr)).copy()
    x = np.abs(rng.normal(1.0, 1.0, (N, t.n)))
    y = rng.normal(0.0, 20.0, (N, t.m))
    return cp, rp, x, y


def _check(t, cp, rp, x, y, status, **perm):
    import harness_sens as H
    got = H.run(t, cp, rp, status, x, y, **perm)
    ref = SN.sensitivities(t, cp, rp, x, y, status)
    sc = SN.scales(t, cp, rp, x, y)
    for g, r, s, what in zip(got, ref, sc, ("rc", "d_cparams", "d_rparams")):
        err = SN.rel_err(g, r, s)
        assert err <= EMU_REL, (what, err)
    return got, ref


@needs_gxx
def test_band_template_in_finalize_order():
    t = TP.wind_battery(24)
    cp, rp, x, y = _inputs(t, 5, 0)
    _check(t, cp, rp, x, y, np.zeros(5, np.int32))


@needs_gxx
def test_csr_template_with_permuted_rows_and_columns():
    t = TP.wind_battery_pem(24)
    rng = np.random.default_rng(1)
    fin = np.flatnonzero(np.isfinite(t.u0)); inf = np.flatnonzero(~np.isfinite(t.u0))
    col_perm = np.concatenate([rng.permutation(fin), rng.permutation(inf)])
    row_perm = rng.permutation(t.m)
    cp, rp, x, y = _inputs(t, 4, 2)
    _check(t, cp, rp, x, y, np.zeros(4, np.int32), col_perm=col_perm, row_perm=row_perm)


@needs_gxx
def test_band_template_with_matrix_params():
    t = TP.wind_battery_design_free_wind(24, None)
    assert t.amap is not None and len(t.amap[0]) > 0
    cp, rp, x, y = _inputs(t, 4, 3)
    rng = np.random.default_rng(4)
    fin = np.flatnonzero(np.isfinite(t.u0)); inf = np.flatnonzero(~np.isfinite(t.u0))
    _check(t, cp, rp, x, y, np.zeros(4, np.int32), col_perm=np.concatenate([rng.permutation(fin), inf]), row_perm=rng.permutation(t.m))


@needs_gxx
def test_dense_template_with_matrix_params():
    t = TP.solar_battery_hydrogen_design(24, None)
    assert t.amap is not None and len(t.amap[0]) > 0
    cp, rp, x, y = _inputs(t, 3, 5)
    fin = np.flatnonzero(np.isfinite(t.u0)); inf = np.flatnonzero(~np.isfinite(t.u0))
    _check(t, cp, rp, x, y, np.zeros(3, np.int32), col_perm=np.concatenate([fin, inf]))     # dense: bounded first, rows kept


@needs_gxx
def test_nan_rows_for_non_optimal_status_and_broadcast_rparams():
    t = TP.wind_battery(24)
    cp, rp, x, y = _inputs(t, 6, 6)
    status = np.array([0, 1, 0, 2, 3, 0], np.int32)
    got, _ = _check(t, cp, rp[0], x, y, status)          # one rparams row shared by the batch (rparams_stride == 0)
    for a in got:
        assert np.isnan(a[status != 0]).all() and np.isfinite(a[status == 0]).all()


# ----------------------------------------------------------------------------------------------------------------- exact
def _exact_grad(t, cp, rp, e: E.ExactOptimum):
    """the gradient of §1 in Fraction arithmetic from the exact optimum's x*, y* (y* and r* exact up to the rounding of their storage)"""
    Fy = [Fraction(float(v)) for v in e.y]
    Fx = [Fraction(float(v)) for v in e.x]
    c, _, _, _ = t.instantiate(cp, rp)
    A = t.matrix(rp).tocsc()
    r = []
    for j in range(t.n):
        s = Fraction(float(c[j]))
        for p in range(A.indptr[j], A.indptr[j + 1]):
            s -= Fraction(float(A.data[p])) * Fy[A.indices[p]]
        r.append(s)
    Cm, Bm, Um = t.Cmap.tocsc(), t.Bmap.tocsc(), t.Umap.tocsc()
    fin = np.isfinite(t.u0)
    dcp = []
    for q in range(t.Pc):
        s = Fraction(float(t.ocmap[q]))
        for p in range(Cm.indptr[q], Cm.indptr[q + 1]):
            s += Fraction(float(Cm.data[p])) * Fx[Cm.indices[p]]
        dcp.append(s)
    drp = []
    for q in range(t.Pr):
        s = Fraction(float(t.omap[q]))
        for p in range(Bm.indptr[q], Bm.indptr[q + 1]):
            s += Fraction(float(Bm.data[p])) * Fy[Bm.indices[p]]
        for p in range(Um.indptr[q], Um.indptr[q + 1]):
            j = Um.indices[p]
            if fin[j]:
                s += Fraction(float(Um.data[p])) * min(r[j], Fraction(0))
        drp.append(s)
    return [float(v) for v in r], np.array([float(v) for v in dcp]), np.array([float(v) for v in drp])


def test_mirror_matches_exact_gradients_on_real_lps():
    s = R.c2(8)
    for k in range(len(s)):
        e = E.exact_optimum(s.t, s.cparams[k], s.rparams[k])
        r, dc, dr = _exact_grad(s.t, s.cparams[k], s.rparams[k], e)
        mr, mdc, mdr = SN.sensitivities(s.t, s.cparams[k][None], s.rparams[k][None], e.x[None], e.y[None])
        sr, sdc, sdr = SN.scales(s.t, s.cparams[k][None], s.rparams[k][None], e.x[None], e.y[None])
        assert SN.rel_err(mr[0], r, sr[0]) < 1e-14
        assert SN.rel_err(mr[0], e.r, sr[0]) < 1e-14          # the certifier's own r* = c - A'y*
        assert SN.rel_err(mdc[0], dc, sdc[0]) < 1e-14
        assert SN.rel_err(mdr[0], dr, sdr[0]) < 1e-14


def one_sided(t, cp, rp, which, q, h0):
    """(left, right) difference quotients of the exact optimal value in parameter q of cparams / rparams: the first step h = h0 / 2^k
    at which the quotients at h and 2h agree on both sides (no breakpoint of the piecewise-linear value inside the step)"""
    f = lambda c, r: E.exact_optimum(t, c, r).obj
    f0 = f(cp, rp)

    def at(d):
        c, r = cp.copy(), rp.copy()
        (c if which == "c" else r)[q] += d
        return f(c, r)
    h = h0
    for _ in range(8):
        q1 = [(at(s * h) - f0) / (s * h) for s in (-1, 1)]
        q2 = [(at(s * 2 * h) - f0) / (s * 2 * h) for s in (-1, 1)]
        if all(abs(a - b) <= 1e-7 * max(1.0, abs(a)) for a, b in zip(q1, q2)):
            return q1[0], q1[1]
        h /= 4
    raise AssertionError("no breakpoint-free step found")


def check_in_interval(g, left, right, convex, tol):
    lo, hi = (left, right) if convex else (right, left)
    assert lo - tol <= g <= hi + tol, (g, left, right, convex)


SUBGRAD_CASES = [
    ("c2", lambda: R.c2(8), [("r", 24), ("r", 5), ("c", 3), ("c", 17)]),
    ("nuclear", lambda: R.nuclear(24, N=4), [("c", 2), ("c", 11)]),
    ("wind_pem", lambda: R.wind_battery_pem(24, N=4), [("r", 24), ("r", 26), ("c", 7)]),
]


@pytest.mark.parametrize("name,make,params", SUBGRAD_CASES, ids=[c[0] for c in SUBGRAD_CASES])
def test_mirror_gradient_lies_between_one_sided_quotients(name, make, params):
    s = make()
    for k in range(min(2, len(s))):
        cp, rp = s.cparams[k].copy(), s.rparams[k].copy()
        _, dc, dr = SN.sensitivities(s.t, cp[None], rp[None] if s.t.Pr else None, s.x[k][None], s.y[k][None])
        for which, q in params:
            if which == "r" and q >= s.t.Pr or which == "c" and q >= s.t.Pc:
                continue
            base = (cp if which == "c" else rp)[q]
            left, right = one_sided(s.t, cp, rp, which, q, 1e-3 * max(1.0, abs(base)))
            g = (dc if which == "c" else dr)[0, q]
            check_in_interval(g, left, right, convex=which == "r", tol=1e-7 * max(1.0, abs(g)))


# ----------------------------------------------------------------------------------------------------------- model space
def test_model_reduced_costs_agree_with_the_template_on_one_to_one_vars():
    """lp_template.model_reduced_costs on the reference-shaped Pyomo wind + battery model (tests/pyomo_stub where Pyomo is absent):
    for every Var that is one template column (lower-bound shifted, boxed or flipped) it equals the template's reduced cost mapped
    through the column scale, the flip and the objective sense; free / presolved Vars get 0; the exact optimum's own r* agrees"""
    from test_pyomo_plugin import PP, build_wind_battery
    from dispatches_b200.lp_template import model_reduced_costs
    T = 24
    lmp, cf, W, P = SC.c2(4)
    m = build_wind_battery(T, lmp[0], cf, W, P)
    t, vars_, cons, p0 = PP.walk_model(m, batch_params=[m.blocks[k].lmp_signal for k in range(T)])
    assert t.meta["recover"]["elim"], "the model's arcs / link equalities are presolved away"
    for k in range(2):
        e = E.exact_optimum(t, lmp[k], lmp[k])
        rc_t, _, _ = SN.sensitivities(t, lmp[k][None], lmp[k][None], e.x[None], e.y[None])
        rcm = model_reduced_costs(t, e.y[None], lmp[k][None])[0]
        rec = t.meta["recover"]
        pos = {nm: q for q, nm in enumerate(t.col_names)}
        sense = t.meta["sense"]
        checked = 0
        scale = np.abs(t.c0).max() + np.abs(e.y).max() * abs(t.A).max()
        for j in range(len(vars_)):
            kind = rec["kind"][j]
            if kind in (1, 2, 4):
                q = pos[rec["names"][rec["col"][j]]]
                want = sense * rec["sgn"][j] * rc_t[0, q] / t.col_scale[q]
                assert rcm[j] == pytest.approx(want, abs=1e-9 * scale), (vars_[j].name, rcm[j], want)
                checked += 1
            elif kind == 3 or kind == 5 and not np.isfinite(vars_[j].lb if vars_[j].lb is not None else -np.inf):
                assert abs(rcm[j]) <= 1e-9 * scale, (vars_[j].name, rcm[j])
        assert checked > 5 * T
