"""The split band kernel (DSP_KERNEL_BAND_SPLIT, dispatches_b200/csrc/dsp_band_split.cuh) on the GPU: planted LPs at every instantiated
half bandwidth against their exact optima, real long-horizon LPs against certified optima, the 25 committed full-year PEM rows, the
band kernel on the same batches, the status rules, the band kernel's retry behind it, its refusals, and x / y in the caller's order."""
import functools
import json
from pathlib import Path

import numpy as np
import pytest

from dispatches_b200 import pricetaker as PT
from dispatches_b200 import scenarios as SC
from dispatches_b200 import solver as S
from dispatches_b200 import templates as TP
from planted_lp import planted, shuffled
from planted_lp import rel as _rel

pytestmark = pytest.mark.gpu

SPLIT = S.KERNEL_BAND_SPLIT
OBJ_REL = 1e-7          # the band kernel's planted-LP bound (tests/test_band_kernel_planted.py)
XY_REL = 1e-6


def _split(t, **kw):
    return S.BatchLPSolver(t, kernel=SPLIT, **kw)


def _solve(sol, cp, rp, **kw):
    n0 = S.launch_count()
    r = sol.solve_host(cp, rp, want_x=True, want_y=True, **kw)
    assert S.launch_count() - n0 == 2          # the split kernel, then the band kernel's retry pass
    ll = S.last_launch()                       # the split kernel's geometry: up to 4 warps per CTA, no shared memory
    assert ll["smem_bytes"] == 0 and 1 <= ll["problems_per_cta"] <= 4 and ll["block"] == 32 * ll["problems_per_cta"], ll
    return r


def _check_planted(p, r, cperm=None, rperm=None, what=""):
    assert (r.status == S.OPTIMAL).all(), (what, r.status, r.iters)
    eo = np.abs(r.obj - p.obj) / np.maximum(1.0, np.abs(p.obj))
    assert eo.max() <= OBJ_REL, (what, eo.max())
    el = np.abs(r.obj - p.obj)[p.lp_mag > 0] / p.lp_mag[p.lp_mag > 0]
    assert el.max(initial=0.0) <= OBJ_REL, (what, el.max())
    x = p.x if cperm is None else p.x[:, cperm]
    y = p.y if rperm is None else p.y[:, rperm]
    if p.unique_x:
        assert _rel(r.x, x) <= XY_REL, what
    if p.unique_y:
        assert _rel(r.y, y) <= XY_REL, what


# (half bandwidth of the planted A A', m): every instantiated W at its minimum m = 64 W, and m not a multiple of 32
PLANTED = [(1, 64), (1, 301), (2, 128), (2, 250), (3, 300), (4, 256), (4, 515), (5, 512), (8, 512), (8, 777)]


@pytest.mark.parametrize("w,m", PLANTED)
def test_planted_lps_reach_their_exact_optima(w, m):
    p = planted(m=m, w=w, seed=3, N=200)
    r = _solve(_split(p.t), p.cparams, p.rparams)
    _check_planted(p, r, what=(w, m))


def test_caller_order_on_a_native_setup_template():
    p = planted(m=300, w=4, seed=9, N=40)
    t, cperm, rperm = shuffled(p.t, seed=7)
    r = _solve(_split(t, native_setup=True), p.cparams, p.rparams)
    _check_planted(p, r, cperm, rperm, "csr_shuffled")


# ------------------------------------------------------------------------------------------------------------------ real LPs
@functools.lru_cache(maxsize=None)
def _pem_set(T, N=4):
    """certified wind + battery + PEM LPs on real T-hour price / capacity-factor windows (tests/real_lps.wind_battery_pem is 24 h)"""
    from real_lps import certify
    p = SC.pool()
    h0 = np.array([500, 2600, 5000, 7100])[:N]
    idx = h0[:, None] + np.arange(T)[None, :]
    cp = np.concatenate([p["dalmp_303"][idx], np.full((N, 1), 2.5)], axis=1)
    rp = TP.wind_battery_rparams(T, p["dacf_303"][idx], SC.FIXED_WIND_MW, 150.0, pem_mw=200.0)
    return certify(TP.wind_battery_pem(T), cp, rp)


def _real(name):
    import real_lps as R
    if name == "nuclear_report_96":
        return R.nuclear_report(96, N=8)
    if name == "fossil_168":
        return R.fossil(168, N=8)
    return _pem_set(168)


@pytest.mark.parametrize("name", ["nuclear_report_96", "fossil_168", "wind_battery_pem_168"])
def test_real_lps_against_certified_optima(name):
    from real_lps import check_exact, fmt
    s = _real(name)
    r = _solve(_split(s.t), s.cparams, s.rparams)
    e = check_exact(s, r.obj, r.status, r.x, r.y, what=name)
    print(name, fmt(e))


# ------------------------------------------------------------------------------------------------------------------ full year
def test_full_year_wind_pem_every_committed_row_through_the_split_kernel():
    """the 25 PEM > 0 rows of the reference's committed wind_PEM_RT_1000 table at T = 8784 through KERNEL_BAND_SPLIT, with the
    tolerances of the band / stage path's test (tests/test_gpu_parity.py)"""
    gold = json.load(open(Path(__file__).parent / "golden" / "wind_pem_golden.json"))["wind_PEM_RT_1000"]
    p = SC.pool()
    fixed = [r for r in range(30) if gold["pem_mw"][r] > 0 and r % 6 != 5]
    design = [r for r in range(30) if r % 6 == 5]
    assert len(fixed) == 20 and len(design) == 5
    n = len(fixed)
    params = {"wind_mw": 847.0, "batt_mw": 0.0, "pem_mw": np.array([gold["pem_mw"][r] for r in fixed]),
              "h2_price_per_kg": np.array([gold["h2_price_per_kg"][r] for r in fixed]), "design_opt": False,
              "extant_wind": True, "wind_resource": np.tile(p["pq1000_rt_cf"], (n, 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (n, 1))}
    res = PT.wind_battery_pem_optimize(8784, params, kernel=SPLIT)
    assert (res.status == S.OPTIMAL).all()
    for k, r in enumerate(fixed):
        scale = TP.PEM_CAP_COST * gold["pem_mw"][r] * 1e3 + TP.PA * (res.annual_rev_h2[k] + abs(res.annual_elec_revenue[k]))
        assert res.NPV[k] == pytest.approx(gold["NPV"][r], rel=2e-7, abs=1e-7 * scale), r
        assert res.annual_rev_h2[k] == pytest.approx(gold["annual_rev_h2"][r], rel=1e-6), r
    n = len(design)
    params.update({"pem_mw": 355.0, "h2_price_per_kg": np.array([gold["h2_price_per_kg"][r] for r in design]), "design_opt": "PEM",
                   "wind_resource": np.tile(p["pq1000_rt_cf"], (n, 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (n, 1))})
    res = PT.wind_battery_pem_optimize(8784, params, kernel=SPLIT)
    assert (res.status == S.OPTIMAL).all()
    for k, r in enumerate(design):
        assert res.sizes["pem_kw"][k] * 1e-3 == pytest.approx(gold["pem_mw"][r], abs=0.06), r
        assert res.NPV[k] == pytest.approx(gold["NPV"][r], rel=1e-6), r


# ------------------------------------------------------------------------------------------------------------------ vs band kernel
def _batches():
    p = SC.pool()
    out = {}
    T = 672
    h0 = 97 * np.arange(24) + 13
    idx = h0[:, None] + np.arange(T)[None, :]
    out["wind_battery_pem_672"] = (TP.wind_battery_pem(T), np.concatenate([p["dalmp_303"][idx], np.full((24, 1), 2.5)], axis=1),
                                   TP.wind_battery_rparams(T, p["dacf_303"][idx], SC.FIXED_WIND_MW, 150.0, pem_mw=200.0))
    out["fossil_168"] = (TP.fossil_surrogate(168), SC.c4(300), None)
    lam = p["nuc_report_lmp_rt"]
    cp = np.stack([np.concatenate([lam[h:h + 672], [1.5]]) for h in 150 * np.arange(24)])
    rp = np.tile([120.0, 20000.0, 20.0], (24, 1))
    out["nuclear_report_672"] = (TP.nuclear_report(672), cp, rp)
    T = 336
    idx = h0[:, None] + np.arange(T)[None, :]
    out["wind_battery_336"] = (TP.wind_battery(T), p["dalmp_303"][idx],
                               TP.wind_battery_rparams(T, p["dacf_303"][idx], SC.FIXED_WIND_MW, 0.25 * SC.FIXED_WIND_MW))
    return out


@pytest.mark.parametrize("name", ["wind_battery_pem_672", "fossil_168", "nuclear_report_672", "wind_battery_336"])
def test_same_status_and_objectives_as_the_band_kernel(name):
    """on a template with a stage descriptor (wind_battery) the split kernel runs as on any band template"""
    t, cp, rp = _batches()[name]
    sp = _split(t)
    r = _solve(sp, cp, rp)
    b = S.BatchLPSolver(t, kernel=S.KERNEL_BAND).solve_host(cp, rp)
    assert np.array_equal(r.status, b.status), (r.status, b.status)
    ok = r.status == S.OPTIMAL
    assert ok.all()
    e = np.abs(r.obj - b.obj) / np.maximum(1.0, np.abs(b.obj))
    assert e.max() <= 1e-9, e.max()
    print(name, "iterations split / band: mean %.1f / %.1f, max %d / %d, obj rel %.1e" % (r.iters.mean(), b.iters.mean(), r.iters.max(),
                                                                                          b.iters.max(), e.max()))


# ------------------------------------------------------------------------------------------------------------------ status rules
N = 8
BAD = 3


def _pem_batch(T=168):
    p = SC.pool()
    starts = 37 * np.arange(N) + 11
    idx = starts[:, None] + np.arange(T)[None, :]
    cp = np.concatenate([p["dalmp_303"][idx], np.full((N, 1), 2.5)], axis=1)
    rp = TP.wind_battery_rparams(T, p["dacf_303"][idx], SC.FIXED_WIND_MW, 150.0, pem_mw=200.0)
    return TP.wind_battery_pem(T), cp, rp


def _rows_equal(r, ref, keep):
    for a, b in ((r.obj[keep], ref.obj), (r.status[keep], ref.status), (r.iters[keep], ref.iters), (r.x[keep], ref.x), (r.y[keep], ref.y)):
        assert np.array_equal(a, b, equal_nan=True)


def test_negative_bound_is_infeasible():
    t, cp, rp = _pem_batch()
    keep = np.array([k for k in range(N) if k != BAD])
    sol = _split(t)
    rpb = rp.copy()
    rpb[BAD, 168] = -5e3            # battery -5 MW (rparams: [wind kW * cf (T) | battery kW | wind kW | PEM kW])
    out = S.LPResult(np.full(N, 12345.0), np.full(N, 7, np.int32), np.full(N, 7, np.int32), np.full((N, t.n), 12345.0),
                     np.full((N, t.m), 12345.0))
    r = _solve(sol, cp, rpb, out=out)
    assert r.status[BAD] == S.INFEASIBLE and np.isnan(r.obj[BAD]) and r.iters[BAD] == 0
    assert np.isnan(r.x[BAD]).all() and np.isnan(r.y[BAD]).all()
    assert (r.status[keep] == S.OPTIMAL).all()
    _rows_equal(r, _solve(sol, cp[keep], rp[keep]), keep)


def test_nan_and_inf_price_leave_the_neighbours_alone():
    t, cp, rp = _pem_batch()
    keep = np.array([k for k in range(N) if k != BAD])
    sol = _split(t)
    ref = _solve(sol, cp[keep], rp[keep])
    for v in (np.nan, np.inf):
        cpn = cp.copy()
        cpn[BAD, 50] = v
        r = _solve(sol, cpn, rp)
        assert r.status[BAD] == S.NUMERICAL, (v, r.status[BAD])
        _rows_equal(r, ref, keep)


def test_iteration_cap_counts_both_attempts_and_the_retry_overwrites_only_non_optimal_lps():
    t, cp, rp = _pem_batch()
    for cap in (3, 14):
        r = _solve(_split(t, max_iter=cap), cp, rp)
        b = S.BatchLPSolver(t, kernel=S.KERNEL_BAND, max_iter=cap).solve_host(cp, rp, want_x=True, want_y=True)
        bad = r.status != S.OPTIMAL
        # what the split kernel left non-optimal is the band kernel's result, bit for bit
        for a, c in ((r.obj, b.obj), (r.status, b.status), (r.iters, b.iters), (r.x, b.x), (r.y, b.y)):
            assert np.array_equal(a[bad], c[bad], equal_nan=True)
        assert (r.iters[bad] == 2 * cap).all()
        if cap == 3:
            assert bad.all()
    r = _solve(_split(t), cp, rp)
    assert (r.status == S.OPTIMAL).all()


# ------------------------------------------------------------------------------------------------------------------ refusals
def _refused(sol, cp, rp, match):
    with pytest.raises(RuntimeError, match=match):
        sol.solve_host(cp, rp)


def test_refusals():
    p = planted(m=63, w=1, seed=1, N=2)              # m < 64 w
    _refused(_split(p.t), p.cparams, p.rparams, r"\(-1\).*needs m >= 64 w")
    p = planted(m=1100, w=16, seed=1, N=2)           # w = 16: not instantiated
    _refused(_split(p.t), p.cparams, p.rparams, r"\(-1\).*half bandwidths up to 8")
    p = planted(m=300, w=4, seed=1, N=2, amap=True)  # per-problem matrix coefficients
    _refused(_split(p.t), p.cparams, p.rparams, r"\(-1\).*does not take per-problem matrix coefficients")
    p = planted(m=300, w=40, seed=1, N=2)            # dense and dense-cluster templates
    for kern, what in ((S.KERNEL_DENSE, "dense kernel"), (S.KERNEL_DENSE_CLUSTER, "dense cluster kernel")):
        sol = S.BatchLPSolver(p.t, kernel=kern)
        sol.opts.kernel = SPLIT
        _refused(sol, p.cparams, p.rparams, rf"\(-1\).*runs only the {what}")
