"""Per-problem matrix coefficients on the dense kernel (dsp_lp_template_create_dense_with_matrix_params): planted LPs whose every
member has its own A, bitwise agreement with the baked-matrix template, the PV + battery + hydrogen design LP with a PV and a reserve
series per scenario against HiGHS and against one-series calls, the status of a non-finite matrix parameter, and the C ABI's
refusals."""
import ctypes as C
import functools
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from dispatches_b200 import pricetaker as PT
from dispatches_b200 import solver as S
from dispatches_b200 import templates as TP
from oracle import highs as H, lp_models as L
from planted_lp import planted, rel

pytestmark = pytest.mark.gpu

GOLD = json.load(open(Path(__file__).parent / "golden" / "solar_golden.json"))
LMP = np.array(GOLD["lmp_24"])
OBJ_REL = 1e-7
XY_REL = 1e-6
THREADS = 256                        # kDenseWarps x 32


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@functools.lru_cache(maxsize=None)
def _resident(m, w, full_span):
    """CTAs the per-LP dense kernel keeps resident for this template (the grid of a launch with more LPs than fit)"""
    p = planted(m, w, seed=1, N=1, full_span=full_span, amap=True)
    sol = S.BatchLPSolver(p.t, kernel=S.KERNEL_DENSE)
    sol.solve_host(np.repeat(p.cparams, 8 * _sms(), axis=0), np.repeat(p.rparams, 8 * _sms(), axis=0))
    return S.last_launch()["grid"]


PLANTED = [(65, 40, False), (100, 99, True), (129, 200, False), (200, 64, False), (500, 48, False), (1024, 40, False)]


@pytest.mark.parametrize("m,w,full", PLANTED, ids=[f"m{m}_w{w}" + ("_full" if f else "") for m, w, f in PLANTED])
def test_planted_lps_with_per_lp_matrices(m, w, full):
    pool = planted(m, w, seed=3, N=6, full_span=full, amap=True)
    t = pool.t
    assert t.w > 32 and t.amap is not None and len(t.amap[0]) > 0
    res = _resident(m, w, full)
    N = 2 * res + 5
    k = np.arange(N) % 6
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE)
    assert sol.dense
    r = sol.solve_host(pool.cparams[k], pool.rparams[k], want_x=True, want_y=True)
    ll = S.last_launch()
    assert ll["block"] == THREADS and ll["problems_per_cta"] == 1 and ll["grid"] == res, ll
    assert (r.status == S.OPTIMAL).all(), (r.status, r.iters)
    for j in range(6, N):                                 # every copy of an LP is its first copy, bit for bit
        assert r.obj[j] == r.obj[j % 6] and r.iters[j] == r.iters[j % 6]
        assert np.array_equal(r.x[j], r.x[j % 6]) and np.array_equal(r.y[j], r.y[j % 6])
    r6 = slice(0, 6)
    assert (np.abs(r.obj[r6] - pool.obj) / np.maximum(1.0, np.abs(pool.obj))).max() < OBJ_REL
    c = np.stack([t.instantiate(pool.cparams[i], pool.rparams[i])[0] for i in range(6)])
    lp_part = (c * r.x[r6]).sum(1) - (c * pool.x).sum(1)
    assert (np.abs(lp_part) / np.maximum(1.0, pool.lp_mag)).max() < OBJ_REL
    assert rel(r.x[r6], pool.x) < XY_REL * pool.scale
    assert rel(r.y[r6], pool.y) < XY_REL
    for i in range(6):                                    # primal residual against the LP's own matrix, and the bounds
        _, b, u, _ = t.instantiate(pool.cparams[i], pool.rparams[i])
        x = r.x[i]
        assert np.abs(t.matrix(pool.rparams[i]) @ x - b).max() <= 1e-8 * max(1.0, np.abs(b).max())
        assert x.min() >= -1e-8 * pool.scale and (x - u)[np.isfinite(u)].max(initial=0.0) <= 1e-8 * pool.scale


def _dyadic(a, grid=1024):
    return np.round(np.asarray(a) * grid) / grid


@pytest.mark.parametrize("T", [24, 48])
def test_bitwise_equal_to_the_baked_template(T):
    """every scenario with the same dyadic, strictly positive PV series: the per-problem template's LP is the baked template's LP bit for
    bit, and so are obj, status, iters, x and y"""
    d = L.solar_default_series()
    rng = np.random.default_rng(T + 1)
    N = 64
    cf = np.maximum(_dyadic(np.tile(d["pv_cfs"], T // 24)), 1.0 / 1024)
    reserve = np.full(T, 100.0)
    lmp = np.tile(LMP, T // 24)[None] * rng.lognormal(0, 0.3, (N, T))
    load = 100.0 * rng.uniform(0.7, 1.2, (N, T))
    baked = S.BatchLPSolver(TP.solar_battery_hydrogen_design(T, cf, reserve_mw=reserve), kernel=S.KERNEL_DENSE)
    a = baked.solve_host(lmp, load * 1e3, want_x=True, want_y=True)
    per = S.BatchLPSolver(TP.solar_battery_hydrogen_design(T, None), kernel=S.KERNEL_DENSE)
    b = per.solve_host(lmp, TP.solar_design_rparams(T, load, cf, reserve), want_x=True, want_y=True)
    assert (a.status == S.OPTIMAL).all()
    for f in ("obj", "status", "iters", "x", "y"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def _design_batch(T, N, seed):
    """own price, load, PV and reserve series per scenario (PV on a 1/1024 grid), zero PV hours in some, one all-zero PV series"""
    d = L.solar_default_series()
    rng = np.random.default_rng(seed)
    lmp = np.tile(LMP, T // 24)[None] * rng.lognormal(0, 0.3, (N, T))
    load = 100.0 * rng.uniform(0.7, 1.2, (N, T))
    cfs = _dyadic(np.tile(d["pv_cfs"], T // 24)[None] * rng.uniform(0.5, 1.0, (N, T)))
    cfs[rng.random((N, T)) < 0.1] = 0.0
    cfs[1] = 0.0
    reserve = 100.0 * rng.uniform(0.4, 1.0, (N, T))
    return lmp, load, cfs, reserve


@pytest.mark.parametrize("T,N", [(24, 512), (48, 64)])
def test_design_batches_with_a_pv_series_per_scenario(T, N):
    lmp, load, cfs, reserve = _design_batch(T, N, T)
    p = dict(pv_mw=0.0, turb_mw=0.0, LMP=lmp, load=load, reserve=reserve, pv_resource=cfs)
    n0 = S.launch_count()
    des, df = PT.pv_battery_hydrogen_design_optimize(T, p)
    assert S.launch_count() == n0 + 1                    # the whole batch in one launch
    assert des["status"] == ["optimal"] * N
    rng = np.random.default_rng(T)
    idx = [0, 1] + sorted(rng.choice(np.arange(2, N), 30, replace=False))
    ref = np.array([-H.solve(L.solar_battery_hydrogen_raw(lmp[k], True, dict(pv_mw=0.0, turb_mw=0.0), pv_cfs=cfs[k], load_mw=load[k],
                                                         reserve_mw=reserve[k]))[0] * 1e3 for k in idx])
    err = np.abs(des["NPV"][idx] - ref) / np.abs(ref)
    print(f"T = {T}: {N} LPs, iterations mean {des['iters'].mean():.1f} max {des['iters'].max()}, max rel NPV error {err.max():.1e}")
    assert err.max() < 1e-6
    excess = df["Excess PV [MW]"] + df["Total PV Generation [MW]"]
    assert np.allclose(excess, des["pv_mw"][:, None] * cfs, rtol=1e-12, atol=1e-9)
    # every scenario against a one-series call of the baked path on that scenario
    keys = set(PT._SOLVERS)
    try:
        sizes = ("pv_mw", "batt_mw", "batt_mwh", "pem_mw", "tank_tonH2", "turb_mw")
        for k in range(N):
            one, _ = PT.pv_battery_hydrogen_design_optimize(T, dict(pv_mw=0.0, turb_mw=0.0, LMP=lmp[k], load=load[k], reserve=reserve[k],
                                                                    pv_resource=cfs[k]))
            assert one["status"] == ["optimal"]
            assert abs(des["NPV"][k] - one["NPV"]) <= 1e-9 * abs(one["NPV"]), k
            for s in sizes:
                assert abs(des[s][k] - one[s]) <= 1e-9 * max(1.0, abs(one[s])), (k, s)
    finally:
        for key in set(PT._SOLVERS) - keys:
            PT._SOLVERS.pop(key).close()


def test_non_finite_matrix_parameter():
    """a NaN / infinite matrix parameter ends the LP with the status the band kernel gives the same defect, the neighbours bitwise
    untouched"""
    dense = planted(65, 40, seed=5, N=4, amap=True)
    band = planted(20, 4, seed=5, N=4, amap=True)
    for v in (np.nan, np.inf):
        got = []
        for pool, kernel in ((dense, S.KERNEL_DENSE), (band, S.KERNEL_BAND)):
            sol = S.BatchLPSolver(pool.t, kernel=kernel)
            ref = sol.solve_host(pool.cparams, pool.rparams, want_x=True, want_y=True)
            rp = pool.rparams.copy()
            rp[2, pool.t.amap[2][0]] = v
            r = sol.solve_host(pool.cparams, rp, want_x=True, want_y=True)
            keep = [0, 1, 3]
            assert (ref.status == S.OPTIMAL).all()
            for f in ("obj", "status", "iters", "x", "y"):
                assert np.array_equal(getattr(r, f)[keep], getattr(ref, f)[keep]), (kernel, f)
            got.append(int(r.status[2]))
        assert got[0] == got[1] and got[0] != S.OPTIMAL, (v, got)


def _desc(t):
    A = t.A.tocsr(); A.sort_indices()
    Cm, Bm, Um = t.Cmap.tocsr(), t.Bmap.tocsr(), t.Umap.tocsr()
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    keep = dict(A_ptr=i32(A.indptr), A_idx=i32(A.indices), A_val=f64(A.data), c0=f64(t.c0), b0=f64(t.b0),
                u0=f64(np.where(np.isfinite(t.u0), t.u0, 1e300)), cm_ptr=i32(Cm.indptr), cm_idx=i32(Cm.indices), cm_val=f64(Cm.data),
                bm_ptr=i32(Bm.indptr), bm_idx=i32(Bm.indices), bm_val=f64(Bm.data), um_ptr=i32(Um.indptr), um_idx=i32(Um.indices),
                um_val=f64(Um.data), omap=f64(t.omap), ocmap=f64(t.ocmap))
    p = lambda k: keep[k].ctypes.data_as(C.c_void_p)
    d = S._LpDesc(m=t.m, n=t.n, Pc=t.Pc, Pr=t.Pr, A_ptr=p("A_ptr"), A_idx=p("A_idx"), A_val=p("A_val"),
                  c0=p("c0"), cmap=S._ParamMap(p("cm_ptr"), p("cm_idx"), p("cm_val")),
                  b0=p("b0"), bmap=S._ParamMap(p("bm_ptr"), p("bm_idx"), p("bm_val")),
                  u0=p("u0"), umap=S._ParamMap(p("um_ptr"), p("um_idx"), p("um_val")), o0=float(t.o0), omap=p("omap"), ocmap=p("ocmap"))
    return d, keep


def test_c_abi_refusals():
    lib = S.load_library()
    pool = planted(65, 40, seed=2, N=1, amap=True)
    t = pool.t
    d, keep = _desc(t)
    r0, c0, k0, v0 = (np.ascontiguousarray(a, dt) for a, dt in zip(t.amap, (np.int32, np.int32, np.int32, np.float64)))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    A = t.A.tocsr()
    off = (0, next(j for j in range(t.n) if j not in set(A.indices[A.indptr[0]:A.indptr[1]])))
    h = C.c_void_p()
    create = lib.dsp_lp_template_create_dense_with_matrix_params
    for rows, cols, params, what in (([off[0]], [off[1]], [k0[0]], b"sparsity pattern"), ([t.m], [c0[0]], [k0[0]], b"out of range"),
                                     ([r0[0]], [t.n], [k0[0]], b"out of range"), ([r0[0]], [c0[0]], [t.Pr], b"out of range"),
                                     ([-1], [c0[0]], [k0[0]], b"out of range")):
        ri, ci, pi = (np.array(a, np.int32) for a in (rows, cols, params))
        assert create(C.byref(d), 1, vp(ri), vp(ci), vp(pi), vp(np.ones(1)), C.byref(h)) == -1
        assert what in lib.dsp_lp_last_error(), lib.dsp_lp_last_error()
    # count == 0 is dsp_lp_template_create_dense: the baked template's results
    assert create(C.byref(d), 0, None, None, None, None, C.byref(h)) == 0
    lib.dsp_lp_template_destroy(h)
    # the matrix-parameter entry point of band templates keeps refusing dense templates
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE)
    one = np.zeros(1, np.int32)
    assert lib.dsp_lp_template_set_matrix_params(sol.handle, 1, vp(one), vp(one), vp(one), vp(np.ones(1))) == -1
    assert b"dense template" in lib.dsp_lp_last_error()
    # DSP_KERNEL_DENSE on a band template with matrix parameters keeps refusing
    band = planted(20, 4, seed=2, N=1, amap=True)
    with pytest.raises(RuntimeError, match="per-problem matrix coefficients"):
        S.BatchLPSolver(band.t, kernel=S.KERNEL_DENSE).solve_host(band.cparams, band.rparams)
