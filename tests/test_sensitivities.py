"""GPU tests of the sensitivity post-pass (dsp_lp_sensitivities, csrc/dsp_sens.cuh): the pass on every kernel family's own (x, y)
against the numpy mirror, against exact optima of real LPs, inside the exact one-sided difference quotients of degenerate LPs, against
the committed full-year wind + PEM table, and its plumbing (determinism, placement independence, broadcast rparams, NaN rows, the
argument errors, one launch per call)."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from dispatches_b200 import pricetaker as PT, scenarios as SC, solver as S, templates as TP
import exact_lp as E
import real_lps as R
import sensitivity_numpy as SN
from test_sensitivities_cpu import check_in_interval, one_sided

pytestmark = pytest.mark.gpu

MIRROR_REL = 1e-12
XY_REL = 1e-6          # the exact-optimum bar of the kernels' x and y (tests/test_dense_matrix_params.py)
dev = torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a, float), device=dev)


def _run(sol, cp, rp):
    """solve with x and y, then the post-pass; numpy (status, x, y, rc, d_cparams, d_rparams)"""
    cpt, rpt = _t(cp), _t(rp) if sol.t.Pr else None
    r = sol.solve(cpt, rpt, want_x=True, want_y=True)
    g = sol.sensitivities(cpt, rpt, r)
    h = lambda a: a.cpu().numpy()
    return h(r.status), h(r.x), h(r.y), h(g.rc), h(g.d_cparams), h(g.d_rparams)


def _pv_set():
    s = R.solar_design_pv(24, N=6)
    return s.t, s.cparams, s.rparams


def _free_wind():
    lmp, cf, _, _ = SC.c2(16, seed=3)
    lmp[::2] *= 40.0
    return TP.wind_battery_design_free_wind(24, None), lmp, np.ascontiguousarray(cf - TP.CF_NOMINAL)


def _windows(T, N):
    """N real T-hour windows of the 303 price and wind series (W = 847 MW, battery 0.25 W) on the wind + battery template"""
    p = SC.pool()
    h0 = np.random.default_rng(T).integers(0, len(p["dalmp_303"]) - T, N)
    idx = h0[:, None] + np.arange(T)[None, :]
    return TP.wind_battery(T), p["dalmp_303"][idx], TP.wind_battery_rparams(T, p["dacf_303"][idx], SC.FIXED_WIND_MW, 0.25 * SC.FIXED_WIND_MW)


def _operation(name):
    x = R.operation(name, T=24, N=8)
    return x.t, x.cparams, x.rparams if x.t.Pr else None


def _set(name):
    x = {"c2": lambda: R.c2(16), "nuclear": lambda: R.nuclear(48, N=8), "pem": lambda: R.wind_battery_pem(24, N=8)}[name]()
    return x.t, x.cparams, x.rparams if x.t.Pr else None


FAMILIES = {
    "stage2": lambda: (*_set("c2"), {}),
    "stage2_long": lambda: (*_windows(168, 8), {}),
    "chain1": lambda: (*_set("nuclear"), {}),
    "band_pem": lambda: (*_set("pem"), dict(kernel=S.KERNEL_BAND)),
    "band_csr_pem": lambda: (*_set("pem"), dict(kernel=S.KERNEL_BAND, native_setup=True)),
    "band_split": lambda: (*_windows(672, 4), dict(kernel=S.KERNEL_BAND_SPLIT)),
    "dense_on_band_template": lambda: (*_set("c2"), dict(kernel=S.KERNEL_DENSE)),
    "dense_matrix_params": lambda: (*_pv_set(), dict(kernel=S.KERNEL_DENSE)),
    "dense_cluster_matrix_params": lambda: (*_pv_set(), dict(kernel=S.KERNEL_DENSE_CLUSTER)),
    "band_matrix_params": lambda: (*_free_wind(), {}),
    "band_double_loop_tracker": lambda: (*_operation("wind_battery_tracker"), dict(kernel=S.KERNEL_BAND)),
}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_every_kernel_family_matches_the_mirror(family):
    t, cp, rp, kw = FAMILIES[family]()
    sol = S.BatchLPSolver(t, **kw)
    st, x, y, rc, dc, dr = _run(sol, cp, rp)
    assert (st == S.OPTIMAL).mean() >= 0.75, st
    N = len(st)
    rpb = np.broadcast_to(rp, (N, t.Pr)) if t.Pr else None
    ref = SN.sensitivities(t, cp, rpb, x, y, st)
    sc = SN.scales(t, cp, rpb, x, y)
    for g, r_, s_, what in zip((rc, dc, dr), ref, sc, ("rc", "d_cparams", "d_rparams")):
        assert SN.rel_err(g, r_, s_) <= MIRROR_REL, (family, what, SN.rel_err(g, r_, s_))


def _norm_scales(t, cp, rp, x, y):
    """SN.scales with every |x_j| and |y_i| replaced by the LP's |x|_inf and |y|_inf: the kernels' x and y are accurate relative to
    their norms (tests/real_lps.py::check_exact), so an entry built from small components is only that accurate"""
    nx = np.abs(x).max(1, keepdims=True) * np.ones_like(x)
    ny = np.abs(y).max(1, keepdims=True) * np.ones_like(y)
    return SN.scales(t, cp, rp, nx, ny)


def _exact_check(s, kw={}):
    sol = S.BatchLPSolver(s.t, **kw)
    st, x, y, rc, dc, dr = _run(sol, s.cparams, s.rparams if s.t.Pr else None)
    assert (st == S.OPTIMAL).all()
    rp = s.rparams if s.t.Pr else None
    er, edc, edr = SN.sensitivities(s.t, s.cparams, rp, s.x, s.y)
    sr, sdc, sdr = _norm_scales(s.t, s.cparams, rp, s.x, s.y)
    worst = {}
    for k in range(len(st)):
        if s.unique_x[k]:
            worst["dc"] = max(worst.get("dc", 0.0), SN.rel_err(dc[k], edc[k], sdc[k]))
        if s.unique_y[k]:
            worst["dr"] = max(worst.get("dr", 0.0), SN.rel_err(dr[k], edr[k], sdr[k]))
            worst["rc"] = max(worst.get("rc", 0.0), SN.rel_err(rc[k], er[k], sr[k]))
    assert worst and all(v <= XY_REL for v in worst.values()), worst
    return worst


@pytest.mark.parametrize("name", ["c2", "nuclear"])
def test_against_exact_optima(name):
    """the certified sets with LPs unique in x or y (the wind + PEM and PV design sets have none: their gradients are checked against
    one-sided quotients below and against the mirror above)"""
    s = {"c2": lambda: R.c2(64), "nuclear": lambda: R.nuclear(48, N=16)}[name]()
    _exact_check(s)


DEGENERATE = [
    ("c2", lambda: R.c2(8), [("r", 24), ("r", 25), ("r", 5), ("r", 13), ("c", 3), ("c", 17)], 8),
    ("nuclear", lambda: R.nuclear(24, N=4), [("c", 2), ("c", 11)], 2),
    ("wind_pem", lambda: R.wind_battery_pem(24, N=4), [("r", 24), ("r", 26), ("c", 7)], 2),
]


@pytest.mark.parametrize("name,make,params,nlp", DEGENERATE, ids=[d[0] for d in DEGENERATE])
def test_gpu_gradient_lies_between_exact_one_sided_quotients(name, make, params, nlp):
    s = make()
    sol = S.BatchLPSolver(s.t)
    st, x, y, rc, dc, dr = _run(sol, s.cparams, s.rparams if s.t.Pr else None)
    assert (st[:nlp] == S.OPTIMAL).all()
    rpb = s.rparams if s.t.Pr else None
    _, sdc, sdr = _norm_scales(s.t, s.cparams, rpb, x, y)
    for k in range(nlp):
        cp, rp = s.cparams[k].copy(), s.rparams[k].copy()
        for which, q in params:
            base = (cp if which == "c" else rp)[q]
            left, right = one_sided(s.t, cp, rp, which, q, 1e-3 * max(1.0, abs(base)))
            g = (dc if which == "c" else dr)[k, q]
            scale = (sdc if which == "c" else sdr)[k, q]
            check_in_interval(g, left, right, convex=which == "r", tol=XY_REL * scale + 1e-7 * max(1.0, abs(g)))


def test_full_year_wind_pem_marginal_pem_value_brackets_the_committed_table():
    """NPV is concave in pem_mw: g(p_a) >= (NPV_b - NPV_a) / (p_b - p_a) >= g(p_b) for consecutive committed fixed-size rows of one
    hydrogen price; and at the design_opt="PEM" optimum p*, g(p* - 1 MW) >= -tol, g(p* + 1 MW) <= tol"""
    gold = json.load(open(Path(__file__).parent / "golden" / "wind_pem_golden.json"))["wind_PEM_RT_1000"]
    p = SC.pool()
    fixed = [r for r in range(30) if gold["pem_mw"][r] > 0 and r % 6 != 5]
    n = len(fixed)
    params = {"wind_mw": 847.0, "batt_mw": 0.0, "pem_mw": np.array([gold["pem_mw"][r] for r in fixed]),
              "h2_price_per_kg": np.array([gold["h2_price_per_kg"][r] for r in fixed]), "design_opt": False,
              "extant_wind": True, "wind_resource": np.tile(p["pq1000_rt_cf"], (n, 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (n, 1))}
    res = PT.wind_battery_pem_optimize(8784, params, want_sensitivities=True)
    assert (res.status == S.OPTIMAL).all()
    g = res.marginal_npv["pem_mw"]
    assert set(res.marginal_npv) == {"wind_mw", "batt_mw", "pem_mw", "h2_price_per_kg", "lmp"}
    # the committed NPVs carry the reference solver's tolerance: 1e-6 relative of the NPV per row, over the size step
    checked = 0
    for a, b in zip(range(n - 1), range(1, n)):
        ra, rb = fixed[a], fixed[b]
        if gold["h2_price_per_kg"][ra] != gold["h2_price_per_kg"][rb] or gold["pem_mw"][rb] <= gold["pem_mw"][ra]:
            continue
        dp = gold["pem_mw"][rb] - gold["pem_mw"][ra]
        slope = (gold["NPV"][rb] - gold["NPV"][ra]) / dp
        tol = 1e-6 * (abs(gold["NPV"][ra]) + abs(gold["NPV"][rb])) / dp
        assert g[a] >= slope - tol and slope + tol >= g[b], (ra, rb, g[a], slope, g[b], tol)
        checked += 1
    assert checked >= 8
    design = [r for r in range(30) if r % 6 == 5]
    h2 = np.array([gold["h2_price_per_kg"][r] for r in design])
    pdes = {"pem_mw": 355.0, "h2_price_per_kg": h2, "design_opt": "PEM", "wind_resource": np.tile(p["pq1000_rt_cf"], (len(design), 1)),
            "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (len(design), 1))}
    dres = PT.wind_battery_pem_optimize(8784, {**params, **pdes})
    pstar = dres.sizes["pem_kw"] * 1e-3
    around = {**params, "pem_mw": np.concatenate([pstar - 1.0, pstar + 1.0]), "h2_price_per_kg": np.concatenate([h2, h2]),
              "wind_resource": np.tile(p["pq1000_rt_cf"], (2 * len(design), 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (2 * len(design), 1))}
    ares = PT.wind_battery_pem_optimize(8784, around, want_sensitivities=True)
    assert (ares.status == S.OPTIMAL).all()
    ga = ares.marginal_npv["pem_mw"]
    tol = 1e-6 * np.abs(dres.NPV)           # the solver's tolerance on the NPV, per MW
    nd = len(design)
    assert (ga[:nd] >= -tol).all() and (ga[nd:] <= tol).all(), (ga, tol)


# ----------------------------------------------------------------------------------------------------------- plumbing
def test_determinism_placement_broadcast_and_launch_count():
    s = R.c2(16)
    sol = S.BatchLPSolver(s.t)
    cpt, rpt = _t(s.cparams), _t(s.rparams)
    r = sol.solve(cpt, rpt, want_x=True, want_y=True)
    n0 = S.launch_count()
    g1 = sol.sensitivities(cpt, rpt, r)
    assert S.launch_count() == n0 + 1
    g2 = sol.sensitivities(cpt, rpt, r)
    assert S.launch_count() == n0 + 2
    for a, b in zip((g1.rc, g1.d_cparams, g1.d_rparams), (g2.rc, g2.d_cparams, g2.d_rparams)):
        assert torch.equal(a, b)
    # one LP alone gives the bits it has inside a shuffled batch of 3000 (several LPs per warp slot, many CTAs)
    perm = np.random.default_rng(0).permutation(np.resize(np.arange(16), 3000))
    pt = torch.as_tensor(perm, device=dev)
    big = S.LPResult(r.obj[pt].contiguous(), r.status[pt].contiguous(), r.iters[pt].contiguous(), r.x[pt].contiguous(), r.y[pt].contiguous())
    gb = sol.sensitivities(cpt[pt].contiguous(), rpt[pt].contiguous(), big)
    for k in range(16):
        one = S.LPResult(r.obj[k:k + 1], r.status[k:k + 1], r.iters[k:k + 1], r.x[k:k + 1], r.y[k:k + 1])
        g = sol.sensitivities(cpt[k:k + 1].contiguous(), rpt[k:k + 1].contiguous(), one)
        for j in np.flatnonzero(perm == k)[:3]:
            assert torch.equal(g.rc[0], gb.rc[j]) and torch.equal(g.d_cparams[0], gb.d_cparams[j]) and torch.equal(g.d_rparams[0], gb.d_rparams[j])
    # rparams_stride == 0: all LPs share LP 0's rparams row
    lmp, cf, W, P = SC.c2(32)
    rp1 = TP.wind_battery_rparams(24, cf, W, P)[0]
    rb = sol.solve(_t(lmp), _t(rp1), want_x=True, want_y=True)
    gbc = sol.sensitivities(_t(lmp), _t(rp1), rb)
    gfull = sol.sensitivities(_t(lmp), _t(np.tile(rp1, (32, 1))), rb)
    assert torch.equal(gbc.d_rparams, gfull.d_rparams) and torch.equal(gbc.rc, gfull.rc)


def test_nan_rows_for_infeasible_and_max_iter():
    lmp, cf, W, P = SC.c2(8)
    rp = np.tile(TP.wind_battery_rparams(24, cf, W, P), (8, 1))
    rp[2, 24] = -1000.0                     # negative battery size through Umap: INFEASIBLE
    sol = S.BatchLPSolver(TP.wind_battery(24))
    st, x, y, rc, dc, dr = _run(sol, lmp, rp)
    assert st[2] == S.INFEASIBLE and (np.delete(st, 2) == S.OPTIMAL).all()
    for a in (rc, dc, dr):
        assert np.isnan(a[2]).all() and np.isfinite(np.delete(a, 2, axis=0)).all()
    short = S.BatchLPSolver(TP.wind_battery(24), max_iter=2)
    st, x, y, rc, dc, dr = _run(short, lmp, TP.wind_battery_rparams(24, cf, W, P)[0])
    assert (st == S.MAX_ITER).all()
    for a in (rc, dc, dr):
        assert np.isnan(a).all()


def test_argument_errors():
    s = R.c2(4)
    sol = S.BatchLPSolver(s.t)
    lib = sol.lib
    cpt, rpt = _t(s.cparams), _t(s.rparams)
    r = sol.solve(cpt, rpt, want_x=True, want_y=True)
    out = torch.empty((4, s.t.n), dtype=torch.float64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    call = lambda N, cp, rp, status, x, y: lib.dsp_lp_sensitivities(sol.handle, N, cp, rp, s.t.Pr, status, x, y, out.data_ptr(), None, None,
                                                                    C.c_void_p(st))
    P = lambda a: a.data_ptr()
    n0 = S.launch_count()
    for args, msg in [((4, P(cpt), P(rpt), None, P(r.x), P(r.y)), b"status"), ((4, P(cpt), P(rpt), P(r.status), None, P(r.y)), b"x"),
                      ((4, P(cpt), P(rpt), P(r.status), P(r.x), None), b"y"), ((-1, P(cpt), P(rpt), P(r.status), P(r.x), P(r.y)), b"N < 0"),
                      ((4, P(cpt), None, P(r.status), P(r.x), P(r.y)), b"rparams")]:
        assert call(*args) == -1
        assert msg in lib.dsp_lp_last_error()
    assert call(0, P(cpt), P(rpt), P(r.status), P(r.x), P(r.y)) == 0
    assert S.launch_count() == n0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------ pricetaker keyword
def _quotients(f, h0):
    """(left, right) difference quotients of the scalar function f at 0: the first h = h0 / 4^k at which the quotients at h and 2h agree
    on both sides (no breakpoint of the piecewise-linear optimal value inside the step)"""
    f0 = f(0.0)
    h = h0
    for _ in range(8):
        q1 = [(f(s * h) - f0) / (s * h) for s in (-1, 1)]
        q2 = [(f(s * 2 * h) - f0) / (s * 2 * h) for s in (-1, 1)]
        if all(abs(a - b) <= 1e-7 * max(1.0, abs(a)) for a, b in zip(q1, q2)):
            return q1
        h /= 4
    raise AssertionError("no breakpoint-free step found")


def _right_quotient(f, h0):
    """the right difference quotient at 0, at the first h = h0 / 4^k where it agrees with the one at 2h"""
    f0 = f(0.0)
    h = h0
    for _ in range(8):
        a, b = (f(h) - f0) / h, (f(2 * h) - f0) / (2 * h)
        if abs(a - b) <= 1e-7 * max(1.0, abs(a)):
            return a
        h /= 4
    raise AssertionError("no breakpoint-free step found")


def _npv(t, cp, rp):
    return -1e5 * E.exact_optimum(t, cp, rp).obj


def test_wind_pem_marginal_battery_value_at_zero_battery():
    """batt_mw = 0, the usual wind + PEM sweep: marginal_npv["batt_mw"] is a supergradient of the (concave) NPV at the boundary of
    its domain, so it is at least the exact right quotient -- the value of the first MW of battery, not only its cost"""
    T, N = 24, 4
    lmp, cf, W, _ = SC.c2(N, seed=5)
    lmp = lmp * np.where(np.arange(T) % 12 < 3, 4.0, 1.0)          # price swings a battery can arbitrage
    params = {"wind_mw": W, "batt_mw": 0.0, "pem_mw": 200.0, "h2_price_per_kg": 2.5, "design_opt": False, "extant_wind": True,
              "wind_resource": np.tile(cf, (N, 1)), "DA_LMPs": lmp}
    res = PT.wind_battery_pem_optimize(T, params, want_sensitivities=True)
    assert (res.status == S.OPTIMAL).all()
    base = PT.wind_battery_pem_optimize(T, params)
    assert np.allclose(res.NPV, base.NPV, rtol=1e-7)
    t = TP.wind_battery_pem(T, with_battery=True)
    g = res.marginal_npv["batt_mw"]
    above_cost = 0
    for k in range(N):
        cp = np.r_[lmp[k], 2.5]
        rpf = lambda z: TP.wind_battery_rparams(T, cf, W, z, pem_mw=200.0)[0]
        right = _right_quotient(lambda z: _npv(t, cp, rpf(z)), 1.0)
        tol = XY_REL * (abs(right) + abs(res.NPV[k]))
        assert g[k] >= right - tol, (k, g[k], right)
        cost = -_right_quotient(lambda z: -1e5 * (t.omap @ rpf(z)), 1.0)         # the battery's annualised cost per MW
        above_cost += right > -cost + 1.0
    assert above_cost >= 1                       # the check is not vacuous: a battery earns more than its cost alone shows


def test_wind_battery_marginal_wind_value_and_the_chain_rule():
    """wind_battery_optimize: marginal_npv["wind_mw"] (chain rule through wind_battery_rparams), ["batt_mw"] and ["lmp"] lie in the
    exact one-sided intervals of the NPV (concave in the sizes, convex in the prices)"""
    T, N = 24, 3
    lmp, cf, W, P = SC.c2(N, seed=11)
    params = {"wind_mw": W, "batt_mw": P, "wind_resource": np.tile(cf, (N, 1)), "DA_LMPs": lmp}
    res = PT.wind_battery_optimize(T, params, want_sensitivities=True)
    assert (res.status == S.OPTIMAL).all() and set(res.marginal_npv) == {"wind_mw", "batt_mw", "lmp"}
    t = TP.wind_battery(T)
    for k in range(N):
        for key, f in (("wind_mw", lambda z: _npv(t, lmp[k], TP.wind_battery_rparams(T, cf, W + z, P)[0])),
                       ("batt_mw", lambda z: _npv(t, lmp[k], TP.wind_battery_rparams(T, cf, W, P + z)[0]))):
            left, right = _quotients(f, 1.0)
            g = res.marginal_npv[key][k]
            tol = XY_REL * (abs(left) + abs(right) + 1.0)
            assert right - tol <= g <= left + tol, (key, k, g, left, right)          # concave
        h = int(np.argmax(cf))
        e = np.eye(T)[h]
        left, right = _quotients(lambda z: _npv(t, lmp[k] + z * e, TP.wind_battery_rparams(T, cf, W, P)[0]), 1.0)
        g = res.marginal_npv["lmp"][k, h]
        assert left - XY_REL * (abs(left) + 1.0) <= g <= right + XY_REL * (abs(right) + 1.0), (k, g, left, right)     # convex


def test_nuclear_marginal_obj_in_the_lmp():
    T = 24
    s = R.nuclear(T, N=4)
    res = PT.nuclear_dispatch_optimize(T, s.cparams, want_sensitivities=True)
    assert res.marginal_npv is None and (res.status == S.OPTIMAL).all()
    g = res.marginal_obj["lmp"]
    for k in range(2):
        for h in (2, 11):
            e = np.eye(T)[h]
            left, right = _quotients(lambda z: E.exact_optimum(s.t, s.cparams[k] + z * e, np.zeros(0)).obj, 1.0)
            tol = XY_REL * (abs(left) + abs(right) + 1e-3)
            assert right - tol <= g[k, h] <= left + tol, (k, h, g[k, h], left, right)      # the cost is concave in the prices
