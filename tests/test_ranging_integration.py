"""GPU tests of the ranging entry points: ``want_ranges=True`` of the price-taker cases and the Pyomo plugin's
``options={"ranging": True}``.  Each moves one hour's LMP to an interior point of its range, solves that batch again with the normal
(interior-point) solve, and checks the objective against the linear prediction from the returned vertex's gradient."""
import numpy as np
import pytest

from dispatches_b200 import pricetaker as PT, scenarios as SC, solver as S
import real_lps as R
from test_pyomo_plugin import build_wind_battery, pyo

pytestmark = pytest.mark.gpu

PRED_REL = 1e-9       # re-solved objective against obj + slope * theta, relative to max(1, |obj|)


def _interior(lo, hi, p):
    """a step from p to an interior point of [lo, hi] (half-way to the farther finite end, or 10 max(1, |p|) on an unbounded side)"""
    if np.isinf(hi):
        return 10.0 * max(1.0, abs(p))
    if np.isinf(lo):
        return -10.0 * max(1.0, abs(p))
    return 0.5 * (hi - p) if hi - p >= p - lo else 0.5 * (lo - p)


def _hours(rng_lmp, lmp, k, count=3):
    """hours of LP k whose LMP range is not a single point, widest first"""
    w = rng_lmp[k, :, 1] - rng_lmp[k, :, 0]
    hs = [h for h in np.argsort(-w) if w[h] > 0]
    assert hs, "every hour of the LP sits at a breakpoint"
    return hs[:count]


def _check_wind(optimize, params, T, N, extra=()):
    res = optimize(T, params, want_ranges=True, want_sensitivities=True)
    assert (res.status == S.OPTIMAL).all()
    rg = res.ranges
    assert set(rg) == {"lmp", "wind_mw", "batt_mw"} | set(extra)
    assert rg["lmp"].shape == (N, T, 2) and all(rg[k].shape == (N, 2) for k in rg if k != "lmp")
    lmp = res.lmp
    assert (rg["lmp"][..., 0] <= lmp).all() and (lmp <= rg["lmp"][..., 1]).all()
    assert (rg["wind_mw"][:, 0] <= np.asarray(params["wind_mw"])).all() and (np.asarray(params["wind_mw"]) <= rg["wind_mw"][:, 1]).all()
    base = optimize(T, params)                                   # the interior-point solve: the vertex has the same objective
    assert np.abs(res.obj - base.obj).max() <= PRED_REL * np.maximum(1.0, np.abs(base.obj)).max()
    for k in range(min(N, 2)):
        for h in _hours(rg["lmp"], lmp, k):
            th = _interior(rg["lmp"][k, h, 0], rg["lmp"][k, h, 1], lmp[k, h])
            moved = dict(params, DA_LMPs=lmp.copy())
            moved["DA_LMPs"][k, h] += th
            again = optimize(T, moved)
            pred = res.obj[k] + th * (-res.marginal_npv["lmp"][k, h] * 1e-5)     # NPV = -1e5 obj
            assert abs(again.obj[k] - pred) <= PRED_REL * max(1.0, abs(again.obj[k])), (k, h, th, again.obj[k], pred)
    return res


def test_wind_battery_want_ranges():
    T, N = 24, 4
    lmp, cf, W, P = SC.c2(N, seed=11)
    cfs = np.tile(cf, (N, 1)) * np.linspace(0.8, 1.0, N)[:, None]        # a capacity-factor series per scenario
    params = {"wind_mw": W, "batt_mw": P, "wind_resource": cfs, "DA_LMPs": lmp}
    res = _check_wind(PT.wind_battery_optimize, params, T, N)
    assert (res.ranges["batt_mw"][:, 0] <= P).all() and (P <= res.ranges["batt_mw"][:, 1]).all()
    plain = PT.wind_battery_optimize(T, params)
    assert plain.ranges is None


def test_wind_battery_pem_want_ranges():
    T, N = 24, 4
    lmp, cf, W, _ = SC.c2(N, seed=5)
    params = {"wind_mw": W, "batt_mw": 0.0, "pem_mw": 200.0, "h2_price_per_kg": 2.5, "design_opt": False, "extant_wind": True,
              "wind_resource": np.tile(cf, (N, 1)), "DA_LMPs": lmp}
    res = _check_wind(PT.wind_battery_pem_optimize, params, T, N, extra=("pem_mw", "h2_price_per_kg"))
    rg = res.ranges
    assert (rg["h2_price_per_kg"][:, 0] <= 2.5).all() and (2.5 <= rg["h2_price_per_kg"][:, 1]).all()
    assert (rg["batt_mw"][:, 0] <= 0.0).all() and (rg["pem_mw"][:, 0] <= 200.0).all() and (200.0 <= rg["pem_mw"][:, 1]).all()


def test_nuclear_want_ranges():
    T = 24
    s = R.nuclear(T, N=4)
    res = PT.nuclear_dispatch_optimize(T, s.cparams, want_ranges=True, want_sensitivities=True)
    assert (res.status == S.OPTIMAL).all() and set(res.ranges) == {"lmp"} and res.ranges["lmp"].shape == (4, T, 2)
    lmp = res.lmp
    for k in range(2):
        for h in _hours(res.ranges["lmp"], lmp, k):
            th = _interior(res.ranges["lmp"][k, h, 0], res.ranges["lmp"][k, h, 1], lmp[k, h])
            moved = lmp.copy()
            moved[k, h] += th
            again = PT.nuclear_dispatch_optimize(T, moved)
            pred = res.obj[k] + th * res.marginal_obj["lmp"][k, h]
            assert abs(again.obj[k] - pred) <= PRED_REL * max(1.0, abs(again.obj[k])), (k, h, th, again.obj[k], pred)


def test_plugin_ranging_option():
    T, N = 24, 4
    lmp, cf, W, P = SC.c2(N)
    m = build_wind_battery(T, lmp[0], cf, W, P)
    bp = lambda L: {m.blocks[t].lmp_signal: L[:, t] for t in range(T)}
    res = pyo.SolverFactory("b200ipm").solve(m, batch_params=bp(lmp), options={"ranging": True, "sensitivities": True})
    pr = res.batch["param_ranges"]
    assert pr.shape == (N, T, 2) and (res.batch["status"] == 0).all() and (res.batch["crossover"]["status"] == 0).all()
    assert (pr[..., 0] <= lmp).all() and (lmp <= pr[..., 1]).all()
    for k in range(2):
        for h in _hours(pr, lmp, k):
            th = _interior(pr[k, h, 0], pr[k, h, 1], lmp[k, h])
            moved = lmp.copy()
            moved[k, h] += th
            # the plugin's default tol of 1e-9 leaves the interior-point objective about 1e-9 from the optimum, the size of the bar
            # itself: the re-solve asks for 1e-11
            again = pyo.SolverFactory("b200ipm").solve(m, batch_params=bp(moved), options={"tol": 1e-11, "feas_tol": 1e-11, "max_iter": 100})
            assert again.batch["status"][k] == 0
            pred = res.batch["obj"][k] + th * res.batch["d_params"][k, h]
            got = again.batch["obj"][k]
            assert abs(got - pred) <= PRED_REL * max(1.0, abs(got)), (k, h, th, got, pred)
