"""The dense cluster kernel (dsp_ipm_dense_cluster_kernel: one LP per thread-block cluster, m <= 4096): planted-optimum LPs across the
old 1024-row limit and up to 4096 rows, the single-CTA dense kernel's answers bit for bit where both run, the PV + battery + hydrogen
design LP over 72, 96 and 168 hours (baked and with a PV series per LP) against HiGHS, a year of prices as 52 week-long LPs in one call, the
status rules, DSP_KERNEL_DENSE_CLUSTER on band templates, and the refusals."""
import ctypes as C

import numpy as np
import pytest

from dispatches_b200 import pricetaker as PT
from dispatches_b200 import scenarios as SC
from dispatches_b200 import solver as S
from dispatches_b200 import templates as TP
from oracle import highs as H, lp_models as L
from planted_lp import planted, rel
from test_dense_mirror import _design_batch
from test_design_pv_series import dyadic_cfs

pytestmark = pytest.mark.gpu

OBJ_REL = 1e-7
XY_REL = 1e-6
THREADS = 256
PAR = dict(pv_mw=0.0, turb_mw=0.0)

PLANTED = [(65, 40, False), (1024, 40, False), (1025, 40, False), (1088, 48, False), (2048, 40, False), (2049, 40, False),
           (4096, 40, False)]


@pytest.mark.parametrize("m,w,full", PLANTED, ids=[f"m{m}_w{w}" + ("_denseA" if f else "") for m, w, f in PLANTED])
def test_planted_lps(m, w, full):
    pool = planted(m, w, seed=3, N=6, full_span=full)
    t = pool.t
    assert t.w > 32
    nt = -(-m // 64)
    csize = 4 if nt <= 32 else 8
    N = 200 // csize + 6                                  # more LPs than clusters in flight: clusters take second tickets
    k = np.arange(N) % 6
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE_CLUSTER)
    r = sol.solve_host(pool.cparams[k], pool.rparams[k], want_x=True, want_y=True)
    ll = S.last_launch()
    assert ll["block"] == THREADS and ll["problems_per_cta"] == csize and ll["grid"] % csize == 0, ll
    assert ll["grid"] // csize < N, ll
    assert (r.status == S.OPTIMAL).all(), (r.status, r.iters)
    for j in range(6, N):                                 # every copy of an LP is its first copy, bit for bit
        assert r.obj[j] == r.obj[j % 6] and r.iters[j] == r.iters[j % 6]
        assert np.array_equal(r.x[j], r.x[j % 6]) and np.array_equal(r.y[j], r.y[j % 6])
    r6 = slice(0, 6)
    assert (np.abs(r.obj[r6] - pool.obj) / np.maximum(1.0, np.abs(pool.obj))).max() < OBJ_REL
    assert rel(r.x[r6], pool.x) < XY_REL * pool.scale
    assert rel(r.y[r6], pool.y) < XY_REL
    print(f"m = {m}: cluster of {csize}, {ll['grid'] // csize} clusters, iterations {r.iters[r6]}")
    if m <= 1024:                                         # where the single-CTA kernel runs too: its answers, bit for bit
        d = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE).solve_host(pool.cparams, pool.rparams, want_x=True, want_y=True)
        for what in ("status", "obj", "iters", "x", "y"):
            assert np.array_equal(getattr(d, what), getattr(r, what)[r6]), (what, "differs from the single-CTA kernel")


def _highs(lmp, load, cfs, T):
    return H.solve(L.solar_battery_hydrogen_raw(lmp, True, PAR, pv_cfs=cfs, load_mw=load, reserve_mw=np.full(T, 100.0)))[0]


@pytest.mark.parametrize("T", [72, 96, 168])
def test_design_lp(T):
    """baked PV series and a PV series per LP (per-problem matrix): all OPTIMAL, a sample within 1e-8 of HiGHS; on a dyadic PV grid the
    per-problem template gives the baked template's answers bit for bit"""
    N = 12
    lmp, load, cfs = _design_batch(T, N, 3)
    tb = TP.solar_battery_hydrogen_design(T, cfs, reserve_mw=np.full(T, 100.0), **PAR)
    assert 1024 < tb.m <= 4096 and tb.w > 32
    r = S.BatchLPSolver(tb, kernel=S.KERNEL_DENSE_CLUSTER).solve_host(lmp, load * 1e3)
    assert (r.status == S.OPTIMAL).all(), (r.status, r.iters)
    idx = [0, 5, 11]
    ref = np.array([_highs(lmp[k], load[k], cfs, T) for k in idx])
    err = np.abs(r.obj[idx] - ref) / np.abs(ref)
    print(f"T = {T} baked: iterations mean {r.iters.mean():.1f} max {r.iters.max()}, max rel error vs HiGHS {err.max():.1e}")
    assert err.max() < 1e-8
    # a PV series per LP
    cf2 = np.stack([dyadic_cfs(T, 10 + k) for k in range(N)])
    tp = TP.solar_battery_hydrogen_design(T, None, **PAR)
    rp = TP.solar_design_rparams(T, load, cf2, np.full((N, T), 100.0))
    sp = S.BatchLPSolver(tp, kernel=S.KERNEL_DENSE_CLUSTER)
    rs = sp.solve_host(lmp, rp, want_x=True)
    assert (rs.status == S.OPTIMAL).all(), (rs.status, rs.iters)
    ref = np.array([_highs(lmp[k], load[k], cf2[k], T) for k in idx])
    err = np.abs(rs.obj[idx] - ref) / np.abs(ref)
    print(f"T = {T} PV series: iterations mean {rs.iters.mean():.1f}, max rel error vs HiGHS {err.max():.1e}")
    assert err.max() < 1e-8
    for k in (0, 7):                                      # the baked template at the same dyadic series: the same bits
        tk = TP.solar_battery_hydrogen_design(T, cf2[k], reserve_mw=np.full(T, 100.0), **PAR)
        rk = S.BatchLPSolver(tk, kernel=S.KERNEL_DENSE_CLUSTER).solve_host(lmp[k:k + 1], load[k:k + 1] * 1e3, want_x=True)
        assert rk.obj[0] == rs.obj[k] and rk.iters[0] == rs.iters[k] and np.array_equal(rk.x[0], rs.x[k])


def test_a_year_in_one_call():
    """52 week-long design LPs of the pool's year of day-ahead prices in one call: all OPTIMAL, NPV within 1e-8 of HiGHS on 4 weeks"""
    lmp = SC.pool()["pq1000_da_lmp"][:8736].reshape(52, 168)
    d = L.solar_default_series()
    cfs = np.tile(d["pv_cfs"], 7)
    p = dict(pv_mw=0.0, turb_mw=0.0, LMP=lmp, load=np.full(168, 100.0), reserve=np.full(168, 100.0), pv_resource=cfs)
    des, _ = PT.pv_battery_hydrogen_design_optimize(168, p, verbose=True)
    assert des["status"] == ["optimal"] * 52, des["iters"]
    assert S.last_launch()["problems_per_cta"] == 8
    weeks = [0, 13, 26, 51]
    ref = np.array([-_highs(lmp[k], np.full(168, 100.0), cfs, 168) * 1e3 for k in weeks])
    err = np.abs(des["NPV"][weeks] - ref) / np.abs(ref)
    print(f"52 weeks: iterations mean {des['iters'].mean():.1f} max {des['iters'].max()}, max rel NPV error vs HiGHS {err.max():.1e}")
    assert err.max() < 1e-8
    with pytest.raises(ValueError, match="m <= 4096"):
        PT.pv_battery_hydrogen_design_optimize(273, {**p, "LMP": np.tile(lmp[0], 2)[:273], "load": np.full(273, 100.0),
                                                     "reserve": np.full(273, 100.0), "pv_resource": np.full(273, 0.5)})


def test_status_rules():
    """a non-finite PV parameter ends that LP NUMERICAL with its neighbours untouched; a negative bound is INFEASIBLE"""
    T, N = 72, 4
    lmp, load, _ = _design_batch(T, N, 5)
    cf2 = np.stack([dyadic_cfs(T, 20 + k) for k in range(N)])
    tp = TP.solar_battery_hydrogen_design(T, None, **PAR)
    rp = TP.solar_design_rparams(T, load, cf2, np.full((N, T), 100.0))
    sol = S.BatchLPSolver(tp, kernel=S.KERNEL_DENSE_CLUSTER)
    ref = sol.solve_host(lmp, rp, want_x=True, want_y=True)
    col = int(tp.amap[2][0])                              # the rparams index of a capacity factor
    bad = rp.copy(); bad[1, col] = np.nan
    r = sol.solve_host(lmp, bad, want_x=True, want_y=True)
    assert r.status[1] == S.NUMERICAL, r.status
    keep = [0, 2, 3]
    assert np.array_equal(r.obj[keep], ref.obj[keep]) and np.array_equal(r.x[keep], ref.x[keep]) and np.array_equal(r.y[keep], ref.y[keep])
    pool = planted(1100, 40, seed=5, N=4)
    t = pool.t
    s2 = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE_CLUSTER)
    j = int(np.flatnonzero(np.isfinite(t.u0))[0])
    c, b, u, _ = t.instantiate(pool.cparams[2], pool.rparams[2])
    row = t.Umap.tocsr()[j]
    rpn = pool.rparams.copy()
    rpn[2, row.indices[0]] -= (u[j] + 5.0) / row.data[0]
    r = s2.solve_host(pool.cparams, rpn, want_x=True)
    assert r.status[2] == S.INFEASIBLE and np.isnan(r.obj[2]) and r.iters[2] == 0 and np.isnan(r.x[2]).all()
    assert (r.status[[0, 1, 3]] == S.OPTIMAL).all()


def _band_sets():
    p = SC.pool()
    rng = np.random.default_rng(11)
    out = {}
    lmp2, cf2, W, P = SC.c2(64)
    out["c2_wind_battery24"] = (TP.wind_battery(24), lmp2, TP.wind_battery_rparams(24, cf2, W, P)[0])
    N = 32
    idx = rng.integers(0, len(p["dalmp_303"]) - 24, N)[:, None] + np.arange(24)[None, :]
    cp = np.concatenate([p["dalmp_303"][idx], np.full((N, 1), 2.5)], axis=1)
    out["pem_cyclic24"] = (TP.wind_battery_pem(24), cp, TP.wind_battery_rparams(24, p["dacf_303"][idx], 200.0, 25.0, pem_mw=25.0))
    T = 512
    s0 = rng.integers(0, len(p["dalmp_303"]) - T, 8)[:, None] + np.arange(T)[None, :]
    out["wind_battery512"] = (TP.wind_battery(T), p["dalmp_303"][s0], TP.wind_battery_rparams(T, p["dacf_303"][:T], 200.0, 25.0)[0])
    return out


@pytest.mark.parametrize("name", ["c2_wind_battery24", "pem_cyclic24", "wind_battery512"])
def test_on_band_templates(name):
    """DSP_KERNEL_DENSE_CLUSTER on a band template: the band kernel's status on every LP, objectives within 3e-11"""
    t, cp, rp = _band_sets()[name]
    band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
    ref = band.solve_host(cp, rp)
    band.opts.kernel = S.KERNEL_DENSE_CLUSTER
    cl = band.solve_host(cp, rp)
    assert S.last_launch()["block"] == THREADS
    assert np.array_equal(cl.status, ref.status), (cl.status, ref.status)
    ok = ref.status == S.OPTIMAL
    err = np.abs(cl.obj[ok] - ref.obj[ok]) / np.maximum(1.0, np.abs(ref.obj[ok]))
    print(f"{name} (m = {t.m}): max rel obj diff {err.max():.1e}")
    assert err.max() < 3e-11


def test_refusals():
    pool = planted(1100, 40, seed=2, N=1)
    sol = S.BatchLPSolver(pool.t, kernel=S.KERNEL_DENSE_CLUSTER)
    for k in (S.KERNEL_BAND, S.KERNEL_STAGE, S.KERNEL_STAGE_V1, S.KERNEL_DENSE):
        sol.opts.kernel = k
        with pytest.raises(RuntimeError, match="only the dense cluster kernel"):
            sol.solve_host(pool.cparams, pool.rparams)
    sol.opts.kernel = S.KERNEL_AUTO
    assert (sol.solve_host(pool.cparams, pool.rparams).status == S.OPTIMAL).all()
    one = np.zeros(1, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    assert sol.lib.dsp_lp_template_set_matrix_params(sol.handle, 1, vp(one), vp(one), vp(one), vp(np.ones(1))) == -1
    assert b"dense template" in sol.lib.dsp_lp_last_error()
    # a band template with per-problem matrix coefficients
    pa = planted(100, 4, seed=1, N=1, amap=True)
    assert pa.t.amap is not None and pa.t.w <= 32
    s2 = S.BatchLPSolver(pa.t)
    s2.opts.kernel = S.KERNEL_DENSE_CLUSTER
    with pytest.raises(RuntimeError, match="DSP_KERNEL_DENSE_CLUSTER does not take per-problem matrix coefficients"):
        s2.solve_host(pa.cparams, pa.rparams)
