"""The dense kernel (dsp_ipm_dense_kernel, csrc/dsp_dense.cuh): planted-optimum LPs whose A A' is wider than the band kernels take
(and with a fully dense A), the same LPs through DSP_KERNEL_DENSE and the usual kernel of band templates, the PV + battery + hydrogen
design LP against the reference's known answer and HiGHS, the status rules, and the refusals."""
import ctypes as C
import functools
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from dispatches_b200 import pricetaker as PT
from dispatches_b200 import scenarios as SC
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
    """CTAs the dense kernel keeps resident for this template (the grid of a launch with more LPs than fit)"""
    p = planted(m, w, seed=1, N=1, full_span=full_span)
    sol = S.BatchLPSolver(p.t, kernel=S.KERNEL_DENSE)
    cp = np.repeat(p.cparams, 8 * _sms(), axis=0)
    rp = np.repeat(p.rparams, 8 * _sms(), axis=0)
    sol.solve_host(cp, rp)
    return S.last_launch()["grid"]


# (m, w, dense A): w > 32 across tile edges, fully dense A, and m = 8 (a band template through DSP_KERNEL_DENSE)
PLANTED = [(8, 8, False), (40, 40, False), (63, 62, True), (64, 64, False), (65, 40, False), (100, 99, True), (129, 200, False),
           (200, 64, False), (500, 48, False), (1024, 40, False)]


@pytest.mark.parametrize("m,w,full", PLANTED, ids=[f"m{m}_w{w}" + ("_denseA" if f else "") for m, w, f in PLANTED])
def test_planted_lps(m, w, full):
    pool = planted(m, w, seed=3, N=6, full_span=full)
    t = pool.t
    if m > 8:
        assert t.w > 32
    res = _resident(m, w, full)
    N = 2 * res + 5
    k = np.arange(N) % 6
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE)
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
    # KKT: primal residual and complementarity of the returned point
    for i in range(6):
        cc, b, u, _ = t.instantiate(pool.cparams[i], pool.rparams[i])
        x = r.x[i]
        assert np.abs(t.A @ x - b).max() <= 1e-8 * max(1.0, np.abs(b).max())
        assert x.min() >= -1e-8 * pool.scale and (x - u)[np.isfinite(u)].max(initial=0.0) <= 1e-8 * pool.scale
    if sol.dense:                                         # a dense template reports the true half bandwidth
        info = (C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32())
        sol.lib.dsp_lp_template_info(sol.handle, *map(C.byref, info))
        assert info[3].value == t.w and info[0].value == t.m


def _cross_sets():
    p = SC.pool()
    rng = np.random.default_rng(11)
    d = L.solar_default_series()
    out = {}
    lmp2, cf2, W, P = SC.c2(64)
    out["c2_wind_battery24"] = (TP.wind_battery(24), lmp2, TP.wind_battery_rparams(24, cf2, W, P)[0], {})
    out["c3_nuclear48"] = (TP.nuclear(48), SC.c3(64), None, {})
    N = 32
    idx = rng.integers(0, len(p["dalmp_303"]) - 24, N)[:, None] + np.arange(24)[None, :]
    cp = np.concatenate([p["dalmp_303"][idx], np.full((N, 1), 2.5)], axis=1)
    out["pem_cyclic24"] = (TP.wind_battery_pem(24), cp, TP.wind_battery_rparams(24, p["dacf_303"][idx], 200.0, 25.0, pem_mw=25.0), {})
    lmp = np.vstack([LMP[None], LMP[None] * rng.lognormal(0, 0.3, (N - 1, 24))])
    out["solar_fixed24"] = (TP.solar_battery_hydrogen(24), lmp, TP.solar_rparams(24, d["pv_cfs"], 200.0, d["load_mw"])[0], {})
    da = p["dalmp_303"][idx]
    rp = TP.wind_battery_operation_rparams(24, p["dacf_303"][idx], 200.0, 25.0, 100.0, rng.uniform(0, 90000, N), rng.uniform(0, 5000, N), None)
    cpb = np.concatenate([da, da * rng.lognormal(0.0, 0.2, (N, 24)), np.full((N, 1), 1e3)], axis=1)
    out["double_loop_bidder24"] = (TP.wind_battery_operation(24, "bidder_da"), cpb, rp, {})
    return out


CROSS = ["c2_wind_battery24", "c3_nuclear48", "pem_cyclic24", "solar_fixed24", "double_loop_bidder24"]


@pytest.mark.parametrize("name", CROSS)
def test_dense_kernel_on_band_templates(name):
    """DSP_KERNEL_DENSE on a band template: the same LPs as its usual kernel -- same status, objectives within 1e-8"""
    t, cp, rp, kw = _cross_sets()[name]
    ref = S.BatchLPSolver(t, **kw).solve_host(cp, rp)
    own = S.last_launch()
    dn = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE, **kw).solve_host(cp, rp)
    ll = S.last_launch()
    assert ll["block"] == THREADS and ll["problems_per_cta"] == 1 and ll != own, ll
    assert np.array_equal(dn.status, ref.status), (dn.status, ref.status)
    ok = ref.status == S.OPTIMAL
    err = np.abs(dn.obj[ok] - ref.obj[ok]) / np.maximum(1.0, np.abs(ref.obj[ok]))
    print(f"{name}: max rel obj diff {err.max():.1e}, iterations dense mean {dn.iters.mean():.2f} vs {ref.iters.mean():.2f}, "
          f"equal on {(dn.iters == ref.iters).mean():.0%}")
    assert err.max() < 1e-8


def _design_params(lmp, load):
    d = L.solar_default_series()
    return dict(pv_mw=0.0, turb_mw=0.0, max_sales=1000, max_purchases=1000, LMP=lmp, load=load, reserve=d["reserve_mw"],
                pv_resource={t: {"pv_resource_config": {"capacity_factor": d["pv_cfs"][t]}} for t in range(24)}, h2_price_per_kg=2.5)


def test_design_lp_reproduces_the_reference():
    d = L.solar_default_series()
    des, df = PT.pv_battery_hydrogen_design_optimize(24, _design_params(LMP, d["load_mw"]))
    assert des["status"] == ["optimal"]
    g = GOLD["test_solar_batt_hydrogen_optimize"]["expect"]
    for k, e in g.items():
        assert des[k] == pytest.approx(e["value"], rel=e.get("rel"), abs=e.get("abs")), k
    assert des["NPV"] == pytest.approx(g["NPV"]["value"], rel=1e-6)
    raw = L.solar_battery_hydrogen_raw(LMP, True, dict(pv_mw=0.0, turb_mw=0.0))
    rep = L.solar_report(raw, H.solve(raw)[1])
    for k in ("batt_mw", "batt_mwh", "capital_cost"):
        assert des[k] == pytest.approx(rep[k], rel=1e-5), k
    out = df["Total Power Output [MW]"] + df["Purchased Power [MW]"] - df["Sold Power [MW]"]
    assert np.abs(out - df["Load [MW]"]).max() < 1e-3
    with pytest.raises(NotImplementedError):
        PT.pv_battery_hydrogen_optimize(24, {**_design_params(LMP, d["load_mw"]), "design_opt": True, "tank_size": 0.0})


@pytest.mark.parametrize("T,N", [(24, 512), (48, 64)])
def test_design_lp_batches_against_highs(T, N):
    d = L.solar_default_series()
    rng = np.random.default_rng(T)
    lmp0 = np.tile(LMP, T // 24)
    lmp = np.vstack([lmp0[None], lmp0[None] * rng.lognormal(0, 0.3, (N - 1, T))])
    load = np.vstack([np.full((1, T), 100.0), 100.0 * rng.uniform(0.7, 1.2, (N - 1, T))])
    cfs = np.tile(d["pv_cfs"], T // 24)
    p = dict(pv_mw=0.0, turb_mw=0.0, LMP=lmp, load=load, reserve=np.full(T, 100.0), pv_resource=cfs)
    des, _ = PT.pv_battery_hydrogen_design_optimize(T, p)
    assert des["status"] == ["optimal"] * N
    idx = [0] + sorted(rng.choice(np.arange(1, N), 31, replace=False))
    ref = np.array([-H.solve(L.solar_battery_hydrogen_raw(lmp[k], True, dict(pv_mw=0.0, turb_mw=0.0), pv_cfs=cfs, load_mw=load[k],
                                                         reserve_mw=np.full(T, 100.0)))[0] * 1e3 for k in idx])
    err = np.abs(des["NPV"][idx] - ref) / np.abs(ref)
    print(f"T = {T}: {N} LPs, iterations mean {des['iters'].mean():.1f} max {des['iters'].max()}, max rel NPV error {err.max():.1e}")
    assert err.max() < 1e-6


def test_status_rules():
    """a negative bound is INFEASIBLE (NaN objective and rows, iters 0) with the neighbours untouched; max_iter = k reports 2k"""
    pool = planted(65, 40, seed=5, N=4)
    t = pool.t
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE)
    ref = sol.solve_host(pool.cparams, pool.rparams, want_x=True, want_y=True)
    rp = pool.rparams.copy()
    j = int(np.flatnonzero(np.isfinite(t.u0))[0])        # a bounded column: its bound comes from the umap terms
    c, b, u, _ = t.instantiate(pool.cparams[2], pool.rparams[2])
    row = t.Umap.tocsr()[j]
    rp[2, row.indices[0]] -= (u[j] + 5.0) / row.data[0]
    r = sol.solve_host(pool.cparams, rp, want_x=True, want_y=True)
    assert r.status[2] == S.INFEASIBLE and np.isnan(r.obj[2]) and r.iters[2] == 0
    assert np.isnan(r.x[2]).all() and np.isnan(r.y[2]).all()
    keep = [0, 1, 3]
    assert np.array_equal(r.obj[keep], ref.obj[keep]) and np.array_equal(r.x[keep], ref.x[keep])
    r = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE, max_iter=3).solve_host(pool.cparams, pool.rparams)
    assert (r.status != S.OPTIMAL).all() and (r.iters == 6).all(), (r.status, r.iters)


def test_status_parity_with_the_band_kernel():
    """the LPs of test_kernel_status_parity (negative and boundary bounds, NaN price, infeasible row): same status as the band kernel"""
    from test_kernel_status_parity import BAD, _family
    for name in ("stage2_T24", "chain_report48"):
        t, cp, rp, kw, ib, icf = _family(name)
        cases = [("nan", cp.copy(), rp)]
        cases[0][1][BAD, 3] = np.nan
        rpb = rp.copy(); rpb[BAD, ib] = -5e3 if name.startswith("stage") else -500.0
        cases.append(("negative", cp, rpb))
        rpz = rp.copy(); rpz[BAD, ib] = -1e-13 * (np.abs(rp[BAD, :icf + 1]).max() if icf is not None else 8000.0)
        cases.append(("boundary", cp, rpz))
        if icf is not None:
            rpi = rp.copy(); rpi[BAD, 0] = -0.1 * np.abs(rp[BAD, :icf + 1]).max()
            cases.append(("infeasible_row", cp, rpi))
        for what, c, r in cases:
            band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND).solve_host(c, r)
            dn = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE).solve_host(c, r)
            assert np.array_equal(dn.status, band.status), (name, what, dn.status, band.status)


def test_refusals():
    big = planted(1100, 40, seed=1, N=1)
    with pytest.raises(RuntimeError, match="m <= 1024"):
        S.BatchLPSolver(big.t, kernel=S.KERNEL_DENSE)
    band_big = planted(1100, 4, seed=1, N=1)
    with pytest.raises(RuntimeError, match="m <= 1024"):
        S.BatchLPSolver(band_big.t, kernel=S.KERNEL_DENSE).solve_host(band_big.cparams, band_big.rparams)
    pool = planted(65, 40, seed=2, N=1)
    sol = S.BatchLPSolver(pool.t, kernel=S.KERNEL_DENSE)
    assert sol.dense
    one = np.zeros(1, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    assert sol.lib.dsp_lp_template_set_matrix_params(sol.handle, 1, vp(one), vp(one), vp(one), vp(np.ones(1))) == -1
    assert b"dense template" in sol.lib.dsp_lp_last_error()
    for k in (S.KERNEL_BAND, S.KERNEL_STAGE, S.KERNEL_STAGE_V1):
        sol.opts.kernel = k
        with pytest.raises(RuntimeError, match="only the dense kernel"):
            sol.solve_host(pool.cparams, pool.rparams)
    sol.opts.kernel = S.KERNEL_AUTO
    assert (sol.solve_host(pool.cparams, pool.rparams).status == S.OPTIMAL).all()
    with pytest.raises(RuntimeError):
        S.BatchLPSolver(pool.t)                    # the plain set-up keeps refusing w > 32
