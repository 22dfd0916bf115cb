"""Parity tests proper: the CUDA solver (through the C-ABI) against the oracle (raw Pyomo-shaped LP + HiGHS)
on the same seeded inputs, plus size-independent certificates at BASELINE.json's full sizes.

Tolerance: north_star asks objective values within 1e-6 relative; the metric is
    |obj_gpu - obj_oracle| / max(1, |obj_oracle|)          (SURVEY.md §8d)
and we additionally bound the error of the LP part alone (objective minus the design-dependent constant)."""
import numpy as np
import pytest
import torch

from dispatches_b200 import pricetaker as PT
from dispatches_b200 import scenarios as SC
from dispatches_b200 import solver as S
from dispatches_b200 import templates as TP
from exact_lp import kkt_residuals
from oracle import highs as H
from oracle import lp_models as L
from planted_stage import KKT_DUAL, KKT_GAP, KKT_PRIMAL

pytestmark = pytest.mark.gpu
REL = 1e-6


def rel_err(a, ref):
    return np.abs(a - ref) / np.maximum(1.0, np.abs(ref))


@pytest.fixture(scope="module")
def wb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    t = TP.wind_battery(24)
    return t, S.BatchLPSolver(t)


def certificate(t, cp, rp, x, y, obj):
    """Size-independent optimality certificate of one solution: objective = c'x + k, and the KKT residuals of (x, y) --
    primal feasibility, dual feasibility of the unbounded columns, duality gap (tests/exact_lp.py)."""
    c, b, u, k = t.instantiate(cp, rp)
    scale = max(1.0, np.abs(b).max())
    assert np.abs(t.A @ x - b).max() <= 1e-7 * scale
    assert x.min() >= -1e-9 * scale and (x - u)[np.isfinite(u)].max() <= 1e-7 * scale
    assert obj == pytest.approx(c @ x + k, rel=1e-9, abs=1e-9)
    kkt = kkt_residuals(t, cp, rp, x, y)
    assert max(kkt["primal"], kkt["bound"]) <= KKT_PRIMAL and kkt["dual_inf"] <= KKT_DUAL and kkt["gap"] <= KKT_GAP, kkt
    return kkt


def test_c1_single_scenario_plumbing(wb):
    t, sol = wb
    lmp, cf, W, P = SC.c1()
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    r = sol.solve_host(lmp[None], rp, want_x=True, want_y=True)
    ref, xref = H.solve(L.wind_battery_raw(lmp, cf, W, P))
    assert r.status[0] == S.OPTIMAL
    assert rel_err(r.obj[0], ref) < REL
    certificate(t, lmp, rp, r.x[0], r.y[0], r.obj[0])


def test_c2_subset_against_oracle(wb):
    t, sol = wb
    lmp, cf, W, P = SC.c2(400)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    r = sol.solve_host(lmp, rp)
    assert (r.status == S.OPTIMAL).all() and r.iters.max() <= 40
    ref, _, _ = H.solve_batch("wind_battery", lmp, kwargs=dict(cf=cf, wind_mw=W, batt_mw=P))
    assert rel_err(r.obj, ref).max() < REL
    k = t.instantiate(lmp[0], rp)[3]
    lp_part = np.abs((r.obj - k) - (ref - k)) / np.maximum(1e-2, np.abs(ref - k))
    assert lp_part.max() < 1e-5


def test_c2_full_batch_certificates(wb):
    """All 10 000 scenarios of BASELINE config 2: every LP optimal, every solution certified."""
    t, sol = wb
    lmp, cf, W, P = SC.c2(10000)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    r = sol.solve_host(lmp, rp, want_x=True, want_y=True)
    assert (r.status == S.OPTIMAL).all()
    assert r.iters.max() <= 40 and 8 <= r.iters.mean() <= 16
    c0, b, u, k = t.instantiate(lmp[0], rp)
    scale = np.abs(b).max()
    # vectorised certificate over the whole batch
    C = (t.Cmap @ lmp.T).T + t.c0
    assert np.abs(r.x @ t.A.T - b).max() <= 1e-7 * scale
    assert r.x.min() >= -1e-9 * scale and (r.x - u)[:, np.isfinite(u)].max() <= 1e-7 * scale
    obj_x = (C * r.x).sum(1) + k
    assert np.allclose(r.obj, obj_x, rtol=1e-9, atol=1e-9)
    rc = C - r.y @ t.A
    ueff = np.where(np.isfinite(u), u, 10.0 * scale)
    lower = r.y @ b + (np.minimum(rc, 0.0) * ueff).sum(1) + k
    gap = (r.obj - lower) / np.maximum(1.0, np.abs(r.obj))
    # the Lagrangian bound multiplies every (rounding-level) negative reduced cost by a 10x-too-large box, so it
    # certifies ~1e-5; the 1e-6 objective parity itself is checked against the oracle in the subset tests.  (It stays here
    # rather than the KKT residuals of certificate(): the batch holds LPs with all-zero prices, c = 0, whose optimal y is 0 and
    # whose returned y is rounding noise, so a duality gap relative to the LP's magnitudes is undefined for them.)
    assert gap.max() <= 2e-5 and gap.min() >= -1e-9


def test_stage_and_band_kernels_agree(wb):
    """Three independent CUDA implementations of the same algorithm: the generic band kernel (shared memory, band LDL'), the
    lane-per-period stage kernel (generation 1: registers, twisted block LDL') and the several-LPs-per-warp stage kernel
    (generation 2: partitioned block elimination) -- same iterates up to the rounding of three elimination orders."""
    t, sol = wb
    assert sol.has_stage
    band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
    v1 = S.BatchLPSolver(t, kernel=S.KERNEL_STAGE_V1)
    lmp, cf, W, P = SC.c2(2000)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    a = sol.solve_host(lmp, rp, want_x=True, want_y=True)
    ll = S.last_launch()
    assert ll["problems_per_cta"] == 4 * (ll["block"] // 32)  # generation 2: four LPs per warp at T = 24
    b = band.solve_host(lmp, rp, want_x=True, want_y=True)
    assert S.last_launch()["smem_bytes"] > 40000
    c = v1.solve_host(lmp, rp, want_x=True, want_y=True)
    assert S.last_launch()["smem_bytes"] == 0                  # generation 1: registers only
    for r in (a, b, c):
        assert (r.status == S.OPTIMAL).all()
    assert rel_err(a.obj, b.obj).max() < 1e-7 and rel_err(a.obj, c.obj).max() < 1e-7
    assert (a.iters == b.iters).mean() > 0.97 and (a.iters == c.iters).mean() > 0.97
    b0 = t.instantiate(lmp[0], rp)[1]
    scale = np.abs(b0).max()
    assert np.abs(a.x @ t.A.T - b0).max() <= 1e-7 * scale
    assert np.abs(a.x - c.x).max() <= 1e-6 * scale and np.abs(a.y - c.y).max() <= 1e-6 * max(1.0, np.abs(c.y).max())


def test_c5_design_sweep_sample_all_optimal(wb):
    """BASELINE config 5 (64 design points x 8760 start hours), strided sample: degenerate hours with zero
    capacity factor and 5 % batteries must still terminate optimal; spot-check against the oracle."""
    t, sol = wb
    lmp, cf, wind, batt = SC.c5()
    sel = np.arange(0, lmp.shape[0], 23)
    rp = TP.wind_battery_rparams(24, cf[sel], wind[sel], batt[sel])
    r = sol.solve_host(lmp[sel], rp)
    assert (r.status == S.OPTIMAL).all(), np.bincount(r.status)
    assert r.iters.max() <= 40
    chk = np.arange(0, sel.size, 211)
    ref = np.array([H.solve(L.wind_battery_raw(lmp[sel[i]], cf[sel[i]], wind[sel[i]], batt[sel[i]]))[0] for i in chk])
    assert rel_err(r.obj[chk], ref).max() < REL


def test_price_scaling_is_linear_in_the_lp_part(wb):
    t, sol = wb
    lmp, cf, W, P = SC.c2(64)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    k = t.instantiate(lmp[0], rp)[3]
    a = sol.solve_host(lmp, rp).obj - k
    b2 = sol.solve_host(2.0 * lmp, rp).obj - k
    assert np.allclose(b2, 2.0 * a, rtol=2e-7, atol=1e-7)


def test_design_batched_rparams(wb):
    """C5-style: capacity factors and sizes differ per LP (rhs / bounds batched)."""
    t, sol = wb
    lmp, cf, wind, batt = SC.c5(3, 3, 24)
    sel = np.arange(0, lmp.shape[0], 7)
    rp = TP.wind_battery_rparams(24, cf[sel], wind[sel], batt[sel])
    r = sol.solve_host(lmp[sel], rp)
    assert (r.status == S.OPTIMAL).all()
    ref = np.array([H.solve(L.wind_battery_raw(lmp[i], cf[i], wind[i], batt[i]))[0] for i in sel])
    assert rel_err(r.obj, ref).max() < REL


def test_edge_cases(wb):
    t, sol = wb
    lmp, cf, W, P = SC.c1()
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    # empty batch
    r0 = sol.solve_host(np.zeros((0, 24)), rp)
    assert r0.obj.shape == (0,)
    # all-zero prices, negative prices, one huge spike, (numerically) no battery
    cases = np.stack([np.zeros(24), -5.0 * np.ones(24), np.where(np.arange(24) == 17, 10000.0, 0.0), lmp])
    r = sol.solve_host(cases, rp)
    assert (r.status == S.OPTIMAL).all()
    ref = np.array([H.solve(L.wind_battery_raw(c, cf, W, P))[0] for c in cases])
    assert rel_err(r.obj, ref).max() < REL
    rp0 = TP.wind_battery_rparams(24, cf, W, 0.0)[0]
    r = sol.solve_host(lmp[None], rp0)
    ref0 = H.solve(L.wind_battery_raw(lmp, cf, W, 0.0))[0]
    assert r.status[0] == S.OPTIMAL and rel_err(r.obj[0], ref0) < REL
    # NaN / infinite prices: NUMERICAL for those LPs only (stage kernel and band kernel), their warp neighbours are unaffected
    bad = np.stack([lmp, lmp, lmp, lmp, 2.0 * lmp])
    bad[1, 5] = np.nan; bad[3, 0] = np.inf
    for solver in (sol, S.BatchLPSolver(t, kernel=S.KERNEL_BAND)):
        r = solver.solve_host(bad, rp)
        assert r.status.tolist() == [S.OPTIMAL, 2, S.OPTIMAL, 2, S.OPTIMAL] and np.isnan(r.obj[[1, 3]]).all()
        assert r.obj[2] == r.obj[0] and rel_err(r.obj[0], ref[3]) < REL


def test_device_and_host_paths_agree_and_count_launches(wb):
    t, sol = wb
    lmp, cf, W, P = SC.c2(300)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    n0 = S.launch_count()
    a = sol.solve_host(lmp, rp)
    dev = torch.device("cuda:0")
    b = sol.solve(torch.tensor(lmp, device=dev), torch.tensor(rp, device=dev))
    torch.cuda.synchronize()
    assert S.launch_count() == n0 + 2
    assert np.array_equal(a.obj, b.obj.cpu().numpy())
    assert np.array_equal(a.iters, b.iters.cpu().numpy())


@pytest.mark.parametrize("with_battery", [True, False])
def test_wind_battery_pem_cyclic_template(with_battery):
    t = TP.wind_battery_pem(24, with_battery=with_battery)
    sol = S.BatchLPSolver(t)
    lmp, cf, W, P = SC.c2(40)
    batt = 150.0 if with_battery else 0.0
    rp = TP.wind_battery_rparams(24, cf, W, batt, pem_mw=200.0)[0]
    cp = np.concatenate([lmp, np.full((40, 1), 2.5)], axis=1)
    r = sol.solve_host(cp, rp)
    assert (r.status == S.OPTIMAL).all()
    ref = np.array([H.solve(L.wind_battery_raw(l, cf, W, batt, pem_mw=200.0, h2_price=2.5))[0] for l in lmp])
    assert rel_err(r.obj, ref).max() < REL


def test_c3_nuclear_subset():
    t = TP.nuclear(48)
    sol = S.BatchLPSolver(t)
    lmp = SC.c3(300)
    r = sol.solve_host(lmp, None)
    assert (r.status == S.OPTIMAL).all()
    ref, _, _ = H.solve_batch("nuclear", lmp)
    assert rel_err(r.obj, ref).max() < REL


def test_c4_fossil_surrogate_subset():
    """Structure-only surrogate: parity against the HiGHS restatement, NOT against the reference's IPOPT NLP."""
    t = TP.fossil_surrogate(168)
    sol = S.BatchLPSolver(t)
    lmp = SC.c4(24)
    r = sol.solve_host(lmp, None)
    assert (r.status == S.OPTIMAL).all()
    ref, _, _ = H.solve_batch("fossil_surrogate", lmp)
    assert rel_err(r.obj, ref).max() < REL


def test_reference_shaped_api():
    """wind_battery_optimize / record_results with the reference's input_params dict."""
    lmp, cf, W, P = SC.c2(16)
    params = {"wind_mw": W, "wind_mw_ub": 10000, "batt_mw": P, "design_opt": False, "extant_wind": True,
              "wind_resource": {t: {"wind_resource_config": {"capacity_factor": [cf[t]]}} for t in range(24)},
              "DA_LMPs": lmp}
    res = PT.wind_battery_optimize(24, params)
    ref = np.array([H.solve(L.wind_battery_raw(l, cf, W, P))[0] for l in lmp])
    assert rel_err(res.obj, ref).max() < REL
    lp = L.wind_battery_raw(lmp[0], cf, W, P)
    rep = L.wind_battery_report(lp, H.solve(lp)[1], lmp[0])
    assert res.NPV[0] == pytest.approx(rep["NPV"], rel=1e-6)
    assert res.annual_revenue[0] == pytest.approx(rep["annual_revenue"], rel=1e-5)
    soc, wind_gen, b2g, w2g, w2b, rev, lmps, wcap, bcap, ann, npv = PT.record_results(res, 0)
    assert len(soc) == 24 and soc[-1] == 0.0 and wcap == pytest.approx(W) and npv == pytest.approx(res.NPV[0])
    # a free wind size with one capacity-factor series per scenario: per-problem matrix coefficients (round 2; refused in round 1)
    cfs = np.stack([cf * (1 - 0.01 * k) for k in range(16)])
    r2 = PT.wind_battery_optimize(24, dict(params, design_opt=True, extant_wind=False, wind_resource=cfs))
    assert (r2.status == S.OPTIMAL).all()
    assert rel_err(r2.obj[5], H.solve(L.wind_battery_raw(lmp[5], cfs[5], W, P, design_opt=True, extant_wind=False))[0]) < REL


def test_sweep_drivers_write_reference_shaped_results(tmp_path):
    """run_design-style sweep: JSON per design point (resume on rerun) and the wind+PEM results table."""
    from dispatches_b200 import run_pricetaker as RP
    lmp, cf, W, P = SC.c2(6)
    out = RP.run_wind_battery_sweep([400.0, 847.0], [0.1, 0.25], lmp, cf, out_dir=tmp_path)
    assert len(out) == 4 and (tmp_path / "result_DA_wind_847.0_battery_0.25.json").exists()
    ref = np.mean([-H.solve(L.wind_battery_raw(l, cf, 847.0, 0.25 * 847.0))[0] * 1e5 for l in lmp])
    assert out[3]["NPV"] == pytest.approx(ref, rel=1e-6)
    n0 = S.launch_count()
    again = RP.run_wind_battery_sweep([400.0, 847.0], [0.1, 0.25], lmp, cf, out_dir=tmp_path)
    assert S.launch_count() == n0 and again == out                       # everything came from the JSON cache
    rows = RP.run_wind_pem_sweep([2.0, 2.5], [0.25, 0.5], lmp, cf, csv_path=tmp_path / "wind_PEM.csv")
    lp = L.wind_battery_raw(lmp[0], cf, 847.0, 0.0, pem_mw=0.25 * 847.0, h2_price=2.0)
    npv = np.mean([-H.solve(L.wind_battery_raw(l, cf, 847.0, 0.0, pem_mw=0.25 * 847.0, h2_price=2.0))[0] * 1e5 for l in lmp])
    assert rows[0]["NPV"] == pytest.approx(npv, rel=1e-6) and (tmp_path / "wind_PEM.csv").exists()


def test_random_designs_and_prices_fuzz(wb):
    """Seeded fuzz over the whole parameter space of the wind+battery template: sizes over two decades, capacity
    factors with exact 0 / 1 hours, negative / zero / spiky prices -- stage kernel vs oracle, all optimal."""
    t, sol = wb
    rng = np.random.default_rng(7)
    N = 240
    pool = SC.pool()
    base = np.concatenate([pool["day_windows"], pool["cluster_days"]])
    lmp = base[rng.integers(0, len(base), N)] * rng.lognormal(0, 0.5, (N, 24))
    lmp[::7] *= -0.3                                   # some negative-price days
    lmp[::11] = 0.0                                    # all-zero days
    cf = rng.beta(0.4, 0.8, (N, 24))
    cf[rng.random((N, 24)) < 0.15] = 0.0
    cf[rng.random((N, 24)) < 0.05] = 1.0
    wind = 10 ** rng.uniform(1.5, 3.7, N)              # 30 MW .. 5 GW
    batt = wind * 10 ** rng.uniform(-2.5, 0.3, N)
    r = sol.solve_host(lmp, TP.wind_battery_rparams(24, cf, wind, batt))
    assert (r.status == S.OPTIMAL).all(), np.bincount(r.status)
    ref = np.array([H.solve(L.wind_battery_raw(lmp[i], cf[i], wind[i], batt[i]))[0] for i in range(N)])
    assert rel_err(r.obj, ref).max() < REL


@pytest.mark.parametrize("T", [2, 5, 7, 12, 13, 23, 31, 32, 33, 48, 49, 96])
def test_stage_kernel_other_horizons(T):
    """Every (lanes per LP, periods per lane) instantiation of the stage kernel -- (2,3) (4,3) (8,3) (16,2) (16,3) (32,3) -- at
    horizons that fill it exactly and that leave periods / lanes idle, against the band kernel and the oracle."""
    t = TP.wind_battery(T)
    stage = S.BatchLPSolver(t, kernel=S.KERNEL_STAGE)
    band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
    p = SC.pool()
    rng = np.random.default_rng(T)
    N = 24
    N = 24 if T <= 32 else 40
    h0 = rng.integers(0, 8000, N)
    idx = h0[:, None] + np.arange(T)[None, :]
    lmp = p["dalmp_303"][idx] * rng.lognormal(0, 0.3, (N, T))
    cf = p["dacf_303"][idx]
    rp = TP.wind_battery_rparams(T, cf, 500.0, 150.0)
    a = stage.solve_host(lmp, rp, want_x=True)
    b = band.solve_host(lmp, rp)
    assert (a.status == S.OPTIMAL).all() and (b.status == S.OPTIMAL).all()
    assert rel_err(a.obj, b.obj).max() < 1e-7
    ref = np.array([H.solve(L.wind_battery_raw(lmp[i], cf[i], 500.0, 150.0))[0] for i in range(0, N, 4)])
    assert rel_err(a.obj[::4], ref).max() < REL
    bb = np.array([t.instantiate(lmp[i], rp[i])[1] for i in range(N)])
    assert np.abs(a.x @ t.A.T - bb).max() <= 1e-7 * np.abs(bb).max()


def test_design_opt_border_column():
    """design_opt=True (battery size is a decision; per-period nameplate columns + link rows, half bandwidth 7, so the
    <8> instantiation of the band kernel): objective and optimal size against the oracle, through the reference API."""
    lmp, cf, W, P = SC.c2(48)
    lmp[::3] *= 40.0                                 # scarcity days make a battery worth building
    t = TP.wind_battery_design(24)
    sol = S.BatchLPSolver(t)
    rp = TP.wind_battery_rparams(24, cf, W, 0.0)[0]
    r = sol.solve_host(lmp, rp, want_x=True)
    assert (r.status == S.OPTIMAL).all(), np.bincount(r.status)
    sols = [H.solve(L.wind_battery_raw(l, cf, W, 0.0, design_opt=True, extant_wind=True)) for l in lmp]
    ref = np.array([s[0] for s in sols])
    assert rel_err(r.obj, ref).max() < REL
    params = {"wind_mw": W, "wind_mw_ub": 10000, "batt_mw": 0.0, "design_opt": True, "extant_wind": True,
              "wind_resource": cf, "DA_LMPs": lmp}
    res = PT.wind_battery_optimize(24, params)
    lp0 = L.wind_battery_raw(lmp[0], cf, W, 0.0, design_opt=True, extant_wind=True)
    p_ref = np.array([s[1][lp0.meta["Bc"]] for s in sols])
    assert p_ref.max() > 1e3                                     # some scenario builds > 1 MW
    big = p_ref > 1e3
    assert np.allclose(res.sizes["batt_kw"][big], p_ref[big], rtol=2e-4)
    assert np.all(res.sizes["batt_kw"][~big] < 1e3 * 1.01 + 50.0)


def test_design_opt_free_wind():
    """design_opt=True with extant_wind=False through the reference-shaped API: wind and battery size are decisions
    (wind_battery_LMP.py:209-219); objective and optimal sizes against the raw oracle LP."""
    lmp, cf, W, P = SC.c2(24)
    scale = np.where(np.arange(24) % 2 == 1, 20.0, 1.0)[:, None]
    ip = {"wind_mw": W, "wind_mw_ub": 10000, "batt_mw": P, "design_opt": True, "extant_wind": False,
          "wind_resource": cf, "DA_LMPs": lmp * scale}
    res = PT.wind_battery_optimize(24, ip)
    assert np.all(res.status == S.OPTIMAL)
    for k in range(0, 24, 3):
        ref, xr = H.solve(L.wind_battery_raw(lmp[k] * scale[k, 0], cf, W, P, design_opt=True, extant_wind=False))
        assert rel_err(res.obj[k], ref) < REL
        raw = L.wind_battery_raw(lmp[k] * scale[k, 0], cf, W, P, design_opt=True, extant_wind=False)
        assert res.sizes["wind_kw"][k] == pytest.approx(xr[raw.meta["Wc"]], rel=1e-4, abs=50.0)


def test_design_opt_free_wind_with_per_scenario_capacity_factors():
    """per-problem MATRIX coefficients (dsp_lp_template_set_matrix_params): design_opt=True, extant_wind=False with a different
    wind series per LMP scenario through the reference-shaped API; objective and optimal sizes against the raw oracle LP."""
    lmp, cf, W, P = SC.c2(48)
    rng = np.random.default_rng(4)
    cfs = np.clip(cf[None, :] * rng.uniform(0.4, 1.6, (48, 24)), 0.0, 1.0)
    scale = np.where(np.arange(48) % 2 == 1, 20.0, 1.0)[:, None]
    ip = {"wind_mw": W, "wind_mw_ub": 10000, "batt_mw": P, "design_opt": True, "extant_wind": False,
          "wind_resource": cfs, "DA_LMPs": lmp * scale}
    res = PT.wind_battery_optimize(24, ip)
    assert np.all(res.status == S.OPTIMAL)
    built = 0
    for k in range(0, 48, 3):
        raw = L.wind_battery_raw(lmp[k] * scale[k, 0], cfs[k], W, P, design_opt=True, extant_wind=False)
        ref, xr = H.solve(raw)
        assert rel_err(res.obj[k], ref) < REL
        assert res.sizes["wind_kw"][k] == pytest.approx(xr[raw.meta["Wc"]], rel=1e-3, abs=100.0)
        built += xr[raw.meta["Wc"]] > 1e3
    assert built >= 3                                  # some scenarios do build wind


def test_design_opt_pem_mode():
    """design_opt="PEM" (run_pricetaker_wind_PEM.py:36-37, pem_ratio None): PEM size optimised, battery fixed at 0."""
    lmp, cf, W, P = SC.c2(40)
    params = {"wind_mw": W, "wind_mw_ub": 10000, "batt_mw": 0.0, "pem_mw": 355.0, "h2_price_per_kg": 2.5,
              "design_opt": "PEM", "extant_wind": True, "wind_resource": cf, "DA_LMPs": lmp}
    res = PT.wind_battery_pem_optimize(24, params)
    assert (res.status == S.OPTIMAL).all()
    sols = [H.solve(L.wind_battery_raw(l, cf, W, 0.0, pem_mw=355.0, h2_price=2.5, design_opt="PEM")) for l in lmp]
    ref = np.array([s[0] for s in sols])
    assert rel_err(res.obj, ref).max() < REL
    lp0 = L.wind_battery_raw(lmp[0], cf, W, 0.0, pem_mw=355.0, h2_price=2.5, design_opt="PEM")
    pem_ref = np.array([s[1][lp0.meta["Pc"]] for s in sols])
    assert np.allclose(res.sizes["pem_kw"], pem_ref, rtol=1e-4, atol=5.0)


def test_full_year_wind_pem_against_the_reference_committed_results():
    """The CUDA path on the reference's own golden: the 8784-period wind+PEM price-taker LPs of
    run_pricetaker_wind_PEM.py (batt_mw = 0) against the committed wind_PEM/wind_PEM_RT_1000.csv NPVs.
    T = 8784 does not fit shared memory: band kernel in global-workspace mode."""
    import json
    from pathlib import Path
    gold = json.load(open(Path(__file__).parent / "golden" / "wind_pem_golden.json"))["wind_PEM_RT_1000"]
    p = SC.pool()
    rows = [1, 4, 8]
    params = {"wind_mw": 847.0, "batt_mw": 0.0, "pem_mw": np.array([gold["pem_mw"][r] for r in rows]),
              "h2_price_per_kg": np.array([gold["h2_price_per_kg"][r] for r in rows]), "design_opt": False,
              "extant_wind": True, "wind_resource": np.tile(p["pq1000_rt_cf"], (3, 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (3, 1))}
    res = PT.wind_battery_pem_optimize(8784, params)
    assert (res.status == S.OPTIMAL).all()
    assert S.last_launch()["smem_bytes"] <= 64                       # workspace mode
    for k, r in enumerate(rows):
        assert res.NPV[k] == pytest.approx(gold["NPV"][r], rel=2e-7)
        assert res.annual_rev_h2[k] == pytest.approx(gold["annual_rev_h2"][r], rel=2e-7)


def test_full_year_wind_pem_every_committed_row_through_the_cuda_path():
    """ALL 25 PEM > 0 rows of the reference's committed wind_PEM/wind_PEM_RT_1000.csv through the CUDA path, two batched calls:
    the 20 fixed-size rows (h2 price and PEM size batched) and the 5 design_opt="PEM" rows (optimal size read back)."""
    import json
    from pathlib import Path
    gold = json.load(open(Path(__file__).parent / "golden" / "wind_pem_golden.json"))["wind_PEM_RT_1000"]
    p = SC.pool()
    fixed = [r for r in range(30) if gold["pem_mw"][r] > 0 and r % 6 != 5]
    design = [r for r in range(30) if r % 6 == 5]
    assert len(fixed) == 20 and len(design) == 5
    n = len(fixed)
    params = {"wind_mw": 847.0, "batt_mw": 0.0, "pem_mw": np.array([gold["pem_mw"][r] for r in fixed]),
              "h2_price_per_kg": np.array([gold["h2_price_per_kg"][r] for r in fixed]), "design_opt": False,
              "extant_wind": True, "wind_resource": np.tile(p["pq1000_rt_cf"], (n, 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (n, 1))}
    res = PT.wind_battery_pem_optimize(8784, params)
    assert (res.status == S.OPTIMAL).all()
    for k, r in enumerate(fixed):
        scale = TP.PEM_CAP_COST * gold["pem_mw"][r] * 1e3 + TP.PA * (res.annual_rev_h2[k] + abs(res.annual_elec_revenue[k]))
        assert res.NPV[k] == pytest.approx(gold["NPV"][r], rel=2e-7, abs=1e-7 * scale), r
        assert res.annual_rev_h2[k] == pytest.approx(gold["annual_rev_h2"][r], rel=1e-6), r
    n = len(design)
    params.update({"pem_mw": 355.0, "h2_price_per_kg": np.array([gold["h2_price_per_kg"][r] for r in design]), "design_opt": "PEM",
                   "wind_resource": np.tile(p["pq1000_rt_cf"], (n, 1)), "DA_LMPs": np.tile(p["pq1000_rt_lmp"], (n, 1))})
    res = PT.wind_battery_pem_optimize(8784, params)
    assert (res.status == S.OPTIMAL).all()
    for k, r in enumerate(design):
        assert res.sizes["pem_kw"][k] * 1e-3 == pytest.approx(gold["pem_mw"][r], abs=0.06), r      # the table rounds to 0.1 MW
        assert res.NPV[k] == pytest.approx(gold["NPV"][r], rel=1e-6), r


def test_c2_full_batch_objective_parity_1e6(wb):
    """BASELINE config C2 in full: all 10 000 objectives within 1e-6 relative of the oracle (HiGHS on the raw LP)."""
    t, sol = wb
    lmp, cf, W, P = SC.c2(10000)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    r = sol.solve_host(lmp, rp)
    assert (r.status == S.OPTIMAL).all()
    ref, _, _ = H.solve_batch("wind_battery", lmp, kwargs=dict(cf=cf, wind_mw=W, batt_mw=P))
    assert rel_err(r.obj, ref).max() < REL


def test_nuclear_report_lp_with_tank_and_turbine_full_year(tmp_path):
    """price_taker_analysis.py:116-222 with tank_capacity / h2_turbine_capacity > 0: the hours couple through the tank holdup, so
    the 8784-period LPs of the enumeration (:353-425) run on the CUDA solver (band kernel, workspace mode) in one batch;
    net NPV against HiGHS on the raw oracle LP, schedule CSVs with the columns of _write_results (:325-350)."""
    import pandas as pd
    from dispatches_b200 import run_pricetaker as RP
    lmp = SC.pool()["nuc_report_lmp_rt"]
    assert lmp.size == 8784
    kw = dict(tank_capacity=50000.0, turbine_capacity=40.0, demand=2000.0)
    res = RP.run_exhaustive_enumeration(lmp, pem_capex=400.0, h2_prices=(1.0, 2.0), pem_fractions=(0.1, 0.3),
                                        schedule_csv_dir=tmp_path, **kw)
    assert all(v == "optimal" for v in res["solver_stat"].values())
    for key, hp, pc in (("00", 1.0, 0.1), ("11", 2.0, 0.3)):
        ref, _ = H.solve(L.nuclear_report_raw(lmp, hp, pc * 400.0, pem_capex=400.0, tank_cap=kw["tank_capacity"],
                                              turbine_cap=kw["turbine_capacity"], demand=kw["demand"]))
        assert res["net_npv"][key] == pytest.approx(-ref / 1e6, rel=1e-6)
    df = pd.read_csv(tmp_path / "results_11_schedule.csv", index_col=0)
    assert list(df.columns) == ["LMP [$/MWh]", "np_to_grid", "np_to_electrolyzer", "tank_holdup_previous", "tank_holdup", "h2_to_pipeline",
                                "h2_to_turbine", "h2_turbine_power", "h2_revenue", "electricity_revenue", "vom", "net_cash_inflow"]
    assert len(df) == 8784 and df["tank_holdup"].max() > 1000.0 and df["tank_holdup"].max() <= 50000.0 * (1 + 1e-6)
    bal = df["tank_holdup"] - df["tank_holdup_previous"] - 20.0 * df["np_to_electrolyzer"] + df["h2_to_pipeline"] + df["h2_to_turbine"]
    assert bal.abs().max() < 1e-3 * 8000.0 * 1e-3


@pytest.mark.parametrize("kind", ["wind_battery", "nuclear", "wind_battery_pem", "bidder_da"])
def test_native_setup_from_plain_csr(kind):
    """dsp_lp_template_create_csr: the library derives column order, row order (RCM vs natural) and the band assembly list itself
    from the plain standard-form LP; results (incl. x and y in the caller's order) equal the Python-prepared descriptor's."""
    if kind == "wind_battery":
        t = TP.wind_battery(24); lmp, cf, W, P = SC.c2(96); cp = lmp; rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    elif kind == "nuclear":
        t = TP.nuclear(48); cp = SC.c3(96); rp = None
    elif kind == "wind_battery_pem":
        t = TP.wind_battery_pem(24); lmp, cf, W, P = SC.c2(96)
        cp = np.concatenate([lmp, np.full((96, 1), 2.5)], axis=1); rp = TP.wind_battery_rparams(24, cf, W, 150.0, pem_mw=200.0)[0]
    else:
        from test_double_loop import CF, G
        t = TP.wind_battery_operation(48, "bidder_da")
        rng = np.random.default_rng(0)
        da = rng.uniform(5, 80, (96, 48)); rt = rng.uniform(5, 80, (96, 48))
        cp = np.concatenate([da, rt, np.full((96, 1), 1e3)], axis=1)
        rp = TP.wind_battery_operation_rparams(48, np.tile(CF, (96, 1)), 200.0, 25.0, 100.0)
    a = S.BatchLPSolver(t, kernel=S.KERNEL_BAND).solve_host(cp, rp, want_x=True, want_y=True)
    b = S.BatchLPSolver(t, kernel=S.KERNEL_BAND, native_setup=True).solve_host(cp, rp, want_x=True, want_y=True)
    assert (a.status == S.OPTIMAL).all() and (b.status == S.OPTIMAL).all()
    assert rel_err(b.obj, a.obj).max() < 1e-8
    scale = max(1.0, np.abs(a.x).max())
    assert np.abs(a.x @ t.A.T - b.x @ t.A.T).max() <= 1e-6 * scale          # same feasible point up to the optimal face


@pytest.mark.parametrize("T", [48, 24, 7, 96])
def test_chain1_stage_kernel_against_band_kernel_and_oracle(T):
    """the descriptor-driven single-storage-chain stage kernel (dsp_stage_chain1.cuh; structure detected on the template) and the
    generic band kernel run the same algorithm: same objectives / iteration counts on the nuclear dispatch LP (C3), x and y in
    template order, and the report's tank / turbine LP with batched capacities."""
    t = TP.nuclear(T)
    a_sol, b_sol = S.BatchLPSolver(t), S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
    assert a_sol.has_chain1 and not b_sol.has_chain1
    p = SC.pool()["cluster_days"]
    rng = np.random.default_rng(T)
    N = 1500
    days = rng.integers(0, len(p) - 4, N)
    lmp = np.stack([np.concatenate([p[k + i] for i in range(4)])[:T] for k in days]) * rng.lognormal(0, 0.25, (N, T))
    a = a_sol.solve_host(lmp, None, want_x=True, want_y=True)
    assert S.last_launch()["block"] % 32 == 0 and S.last_launch()["problems_per_cta"] >= 1
    b = b_sol.solve_host(lmp, None, want_x=True, want_y=True)
    assert (a.status == S.OPTIMAL).all() and (b.status == S.OPTIMAL).all()
    assert rel_err(a.obj, b.obj).max() < 1e-8 and (a.iters == b.iters).mean() > 0.97
    ref = np.array([H.solve(L.nuclear_raw(l))[0] for l in lmp[:24]]) if T == 48 else None
    if ref is not None:
        assert rel_err(a.obj[:24], ref).max() < REL
    c, bb, u, k = t.instantiate(lmp[0], np.zeros(0))
    scale = max(1.0, np.abs(u[np.isfinite(u)]).max())
    assert np.abs(a.x @ t.A.T - bb).max() <= 1e-7 * scale and np.abs(a.y - b.y).max() <= 1e-5 * max(1.0, np.abs(b.y).max())
    if T == 48:
        tr = TP.nuclear_report(T, demand=2000.0)
        sr = S.BatchLPSolver(tr)
        assert sr.has_chain1
        lm = SC.pool()["nuc_report_lmp_rt"][1000:1000 + T]
        cases = [(hp, pem, tank, turb) for hp in (0.75, 1.25, 2.0) for pem in (40.0, 120.0, 200.0) for tank, turb in ((30000.0, 0.0), (50000.0, 40.0), (0.0, 25.0))]
        cp = np.array([np.r_[lm, c_[0]] for c_ in cases]); rp = np.array([[c_[1], c_[2], c_[3]] for c_ in cases])
        r = sr.solve_host(cp, rp)
        refr = np.array([H.solve(L.nuclear_report_raw(lm, hp, pem, pem_capex=400.0, tank_cap=tank, turbine_cap=turb, demand=2000.0))[0]
                         for hp, pem, tank, turb in cases])
        assert (r.status == S.OPTIMAL).all() and rel_err(r.obj, refr).max() < REL


def test_the_c_abi_from_plain_c(tmp_path):
    """INTEGRATION.md 1b: a C program (tests/c_abi_example.c) creates a template from plain CSR, solves a batch, reads x"""
    import subprocess
    from test_cabi import build_c_example
    r = subprocess.run([str(build_c_example(tmp_path))], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "C ABI OK" in r.stdout, r.stdout + r.stderr


def test_long_horizon_wind_battery_quarter_year():
    """run_pricetaker_wind_battery.run_design's kind of LP (the reference uses n_time_points = 8736): a 2184-period
    wind+battery LP against the oracle; the throughput column grows with the horizon (scale-invariant proximal term)."""
    p = SC.pool()
    T = 2184
    lam, cf = p["dalmp_303"][:T], p["dacf_303"][:T]
    par = {"wind_mw": 847.0, "batt_mw": np.array([84.7, 211.75]), "design_opt": False, "extant_wind": True,
           "wind_resource": np.tile(cf, (2, 1)), "DA_LMPs": np.tile(lam, (2, 1))}
    res = PT.wind_battery_optimize(T, par, want_solution=False)
    assert (res.status == S.OPTIMAL).all() and res.iters.max() <= 60
    ref = np.array([H.solve(L.wind_battery_raw(lam, cf, 847.0, b))[0] for b in (84.7, 211.75)])
    assert rel_err(res.obj, ref).max() < REL


def test_full_year_wind_battery_on_the_long_horizon_kernel():
    """the reference's real sweep LP (run_pricetaker_wind_battery.py:57-58: n_time_points = 8736) on the AUTO path: long-horizon stage
    kernel (one warp per LP, partitioned elimination, state in the workspace) with the band kernel re-solving what it leaves
    non-optimal -- against the band kernel alone on every LP and against the oracle on one"""
    import torch
    p = SC.pool()
    T, N = 8736, 8
    t = TP.wind_battery(T)
    lam, cf = p["dalmp_303"][:T], p["dacf_303"][:T]
    wind = np.linspace(200.0, 1600.0, N); batt = wind * np.linspace(0.05, 1.0, N)[::-1]
    rp = torch.tensor(TP.wind_battery_rparams(T, np.tile(cf, (N, 1)), wind, batt), device="cuda")
    cp = torch.tensor(np.tile(lam, (N, 1)), device="cuda")
    auto = S.BatchLPSolver(t).solve(cp, rp)
    band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND).solve(cp, rp)
    torch.cuda.synchronize()
    assert int((auto.status != 0).sum()) == 0 and int((band.status != 0).sum()) == 0
    a, b = auto.obj.cpu().numpy(), band.obj.cpu().numpy()
    assert rel_err(a, b).max() < 1e-8
    ref = H.solve(L.wind_battery_raw(lam, cf, wind[2], batt[2]))[0]
    assert abs(a[2] - ref) / max(1.0, abs(ref)) < REL


def test_determinism_and_permutation_invariance(wb):
    """Size-independent properties at the full C2 size: the ticket dispatcher hands LPs to warps in a run-dependent
    order, yet every LP's result depends on its own data only -- two runs agree bit for bit, and permuting the batch
    permutes the results."""
    t, sol = wb
    lmp, cf, W, P = SC.c2(10000)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    a = sol.solve_host(lmp, rp)
    b = sol.solve_host(lmp, rp)
    assert np.array_equal(a.obj, b.obj) and np.array_equal(a.iters, b.iters) and np.array_equal(a.status, b.status)
    perm = np.random.default_rng(0).permutation(10000)
    c = sol.solve_host(np.ascontiguousarray(lmp[perm]), rp)
    assert np.array_equal(c.obj, a.obj[perm]) and np.array_equal(c.iters, a.iters[perm])
    # checksum of checksums: batch split in two halves solved separately
    d1 = sol.solve_host(np.ascontiguousarray(lmp[:5000]), rp); d2 = sol.solve_host(np.ascontiguousarray(lmp[5000:]), rp)
    assert np.array_equal(np.concatenate([d1.obj, d2.obj]), a.obj)
