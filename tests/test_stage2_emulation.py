"""The generation-2 stage kernel's CUDA SOURCE (dispatches_b200/csrc/dsp_stage2.cuh) executed on CPU lanes: tests/emu compiles
the warp body with g++ on a lock-step SIMT emulator (every shuffle / vote is a 32-lane barrier).  Checks, without a GPU:
the partitioned elimination, the several-LPs-per-warp bookkeeping (group refill from the ticket counter, second attempt,
masking of inactive periods) against the oracle (HiGHS) and the numpy mirror of the algorithm."""
import shutil

import numpy as np
import pytest

from dispatches_b200 import scenarios as SC, templates as TP
from exact_lp import kkt_residuals
from oracle import highs as H, ipm_stage_numpy as M, lp_models as L
from planted_stage import KKT_DUAL, KKT_GAP, KKT_PRIMAL

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


@pytest.fixture(scope="module")
def emu():
    import importlib.util, pathlib
    spec = importlib.util.spec_from_file_location("emu_harness", pathlib.Path(__file__).parent / "emu" / "harness.py")
    harness = importlib.util.module_from_spec(spec); spec.loader.exec_module(harness)
    harness.build()
    return harness


def rel_err(a, ref):
    return np.abs(a - ref) / np.maximum(1.0, np.abs(ref))


def test_c2_sample_matches_oracle_and_mirror(emu):
    t = TP.wind_battery(24)
    st = t.meta["stage_wb"]
    lmp, cf, W, P = SC.c2(150)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    # 150 LPs on 2 warps x 4 groups: every group refills several times, the last tickets leave groups idle
    obj, status, iters, x, y = emu.solve(t, lmp, rp, 8, 3, warps=2)
    assert (status == 0).all()
    ref, _, _ = H.solve_batch("wind_battery", lmp, kwargs=dict(cf=cf, wind_mw=W, batt_mw=P), procs=1)
    assert rel_err(obj, ref).max() < 1e-7
    consts = {k: st[k] for k in ("a", "binv", "half", "delta", "dur", "k_rev")}
    m = M.solve_batch(lmp, rp[:24], rp[24], consts)
    assert np.array_equal(iters, m["iters"])            # same algorithm, another elimination order
    k = t.instantiate(lmp[0], rp)[3]
    assert rel_err(obj, m["obj_lp"] + k).max() < 1e-10
    # primal / dual write-back: the KKT residuals of (x, y) (the exact x and y are checked in test_planted_stage.py)
    c, b, u, k = t.instantiate(lmp[7], rp)
    assert x[7].min() >= -1e-9 * np.abs(b).max()
    assert obj[7] == pytest.approx(c @ x[7] + k, rel=1e-9, abs=1e-9)
    kkt = kkt_residuals(t, lmp[7], rp, x[7], y[7])
    assert max(kkt["primal"], kkt["bound"]) <= KKT_PRIMAL and kkt["dual_inf"] <= KKT_DUAL and kkt["gap"] <= KKT_GAP, kkt


def test_design_sweep_sample_rhs_batched(emu):
    t = TP.wind_battery(24)
    lmp, cf, w, b = SC.c5()
    sel = np.random.default_rng(11).choice(lmp.shape[0], 60, replace=False)
    rp = TP.wind_battery_rparams(24, cf[sel], w[sel], b[sel])
    obj, status, iters, _, _ = emu.solve(t, lmp[sel], rp, 8, 3, warps=3, want_xy=False)
    assert (status == 0).all()
    ref = np.array([H.solve(L.wind_battery_raw(lmp[i], cf[i], w[i], b[i]))[0] for i in sel])
    assert rel_err(obj, ref).max() < 1e-7


@pytest.mark.parametrize("T,Lg,P", [(2, 2, 3), (5, 2, 3), (7, 4, 3), (12, 4, 3), (13, 8, 3), (23, 8, 3), (31, 16, 2), (32, 16, 2),
                                    (33, 16, 3), (48, 16, 3), (49, 32, 3), (96, 32, 3), (20, 32, 1)])
def test_other_horizons_and_geometries(emu, T, Lg, P):
    """every instantiation the library ships (and the lane-per-period limit P = 1), horizons that leave periods / lanes idle"""
    t = TP.wind_battery(T)
    p = SC.pool()
    rng = np.random.default_rng(T)
    N = 9
    starts = rng.integers(0, 8736 - T, N)
    lmp = np.stack([p["dalmp_303"][s:s + T] for s in starts]) * rng.lognormal(0, 0.25, (N, T))
    cfs = np.stack([p["dacf_303"][s:s + T] for s in starts])
    wind, batt = rng.uniform(200, 1600, N), rng.uniform(10, 800, N)
    rp = TP.wind_battery_rparams(T, cfs, wind, batt)
    obj, status, iters, x, _ = emu.solve(t, lmp, rp, Lg, P, warps=2)
    assert (status == 0).all()
    ref = np.array([H.solve(L.wind_battery_raw(lmp[i], cfs[i], wind[i], batt[i]))[0] for i in range(N)])
    assert rel_err(obj, ref).max() < 1e-7
    c, b, u, k = t.instantiate(lmp[0], rp[0])
    assert np.abs(t.A @ x[0] - b).max() <= 1e-7 * np.abs(b).max()


def test_edge_cases(emu):
    t = TP.wind_battery(24)
    lmp, cf, W, P = SC.c2(8)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    cases = np.stack([np.zeros(24), np.full(24, 10000.0), np.r_[np.zeros(23), 10000.0], lmp[0], 1e-6 * lmp[1]])
    obj, status, _, _, _ = emu.solve(t, cases, rp, 8, 3)
    assert (status == 0).all()
    ref = np.array([H.solve(L.wind_battery_raw(c, cf, W, P))[0] for c in cases])
    assert rel_err(obj, ref).max() < 1e-6
    # no battery, and a negative battery size (infeasible bound) next to regular LPs in the same warp
    rps = np.tile(rp, (6, 1))
    rps[1, 24] = 0.0
    rps[4, 24] = -5.0
    obj, status, iters, _, _ = emu.solve(t, lmp[:6], rps, 8, 3)
    assert status[4] == 3 and np.isnan(obj[4]) and (np.delete(status, 4) == 0).all()
    assert obj[1] == pytest.approx(H.solve(L.wind_battery_raw(lmp[1], cf, W, 0.0))[0], rel=1e-7)
    # the second attempt: an iteration cap forces attempt 1 (shorter step, stronger proximal term) and both counts add up
    obj, status, iters, _, _ = emu.solve(t, lmp[:5], rp, 8, 3, max_iter=6)
    assert (status != 0).all() and (iters == 6 + 6).all()
    # NaN / infinite prices end as NUMERICAL without disturbing the LPs that share their warp; all-negative prices are a regular LP
    bad = lmp[:6].copy()
    bad[1, 5] = np.nan; bad[3, 0] = np.inf; bad[4, :] = -50.0
    obj, status, iters, _, _ = emu.solve(t, bad, rp, 8, 3)
    assert status.tolist() == [0, 2, 0, 2, 0, 0] and np.isnan(obj[[1, 3]]).all()
    ref = np.array([H.solve(L.wind_battery_raw(bad[k], cf, W, P))[0] for k in (0, 2, 4, 5)])
    assert rel_err(obj[[0, 2, 4, 5]], ref).max() < 1e-7
    # empty batch and a single LP (three of the four groups never get work)
    obj, status, _, _, _ = emu.solve(t, np.zeros((0, 24)), rp, 8, 3)
    assert obj.size == 0
    obj, status, _, _, _ = emu.solve(t, lmp[:1], rp, 8, 3)
    assert status[0] == 0


@pytest.mark.parametrize("T", [97, 168, 672])
def test_long_horizon_variant(emu, T):
    """dsp_stage2_long.cuh (T > 96: one warp per LP, ceil(T / 32) periods per lane, iterate and temporaries in a workspace):
    the same algorithm with rolled period loops -- against the oracle, with sizes and capacity factors batched."""
    t = TP.wind_battery(T)
    p = SC.pool()
    rng = np.random.default_rng(T)
    N = 3
    starts = rng.integers(0, 8736 - T, N)
    lmp = np.stack([p["dalmp_303"][s:s + T] for s in starts]) * rng.lognormal(0, 0.25, (N, T))
    cfs = np.stack([p["dacf_303"][s:s + T] for s in starts])
    wind, batt = rng.uniform(200, 1600, N), rng.uniform(10, 800, N)
    rp = TP.wind_battery_rparams(T, cfs, wind, batt)
    obj, status, iters, x, y = emu.solve_long(t, lmp, rp, warps=2)
    assert (status == 0).all()
    ref = np.array([H.solve(L.wind_battery_raw(lmp[i], cfs[i], wind[i], batt[i]))[0] for i in range(N)])
    assert rel_err(obj, ref).max() < 1e-7
    c, b, u, k = t.instantiate(lmp[0], rp[0])
    assert np.abs(t.A @ x[0] - b).max() <= 1e-7 * np.abs(b).max()
    assert obj[0] == pytest.approx(c @ x[0] + k, rel=1e-9, abs=1e-9)
