"""GPU tests of ``want_curves`` of the price-taker cases (dsp_lp_parametric through pricetaker): for every curve name of the three cases,
a sample of LPs is solved again at the midpoint of every segment of the curve (and past its last event), and the objective must equal
``curves[name].value(p)``; on the hourly LMP curves the slope of every segment must equal the gradient at the re-solved vertex, i.e.
minus the energy sold in that hour (renewables: in NPV units).  The re-solve is the normal interior-point solve followed by the
crossover (``want_ranges=True``): the interior-point objective alone is about 1e-9 from the optimum at the default tolerance, the size
of the bar itself, while the vertex's is exact to rounding."""
import math

import numpy as np
import pytest

from dispatches_b200 import pricetaker as PT, scenarios as SC, solver as S
import real_lps as R

pytestmark = pytest.mark.gpu

PRED_REL = 1e-9       # re-solved objective against the curve, relative to max(1, |obj|), in the LP's objective units
LPS = 2               # LPs of each batch whose curves are re-solved
HOURS = (2, 13, 20)   # the LMP hours sampled


def _points(curve, idx, end):
    """midpoints of the positive-length segments of curve[idx] up to end, and 10 max(1, |p0|) past the last event of an open end"""
    c, at = int(curve.count[idx]), curve.at[idx]
    if curve.status[idx] in (3, 4):
        c -= 1
    pts = [0.5 * (at[e] + at[e + 1]) for e in range(c - 1) if at[e + 1] > at[e]]
    last = at[c - 1]
    pts.append(last + 10.0 * max(1.0, abs(at[0])) if math.isinf(end) else 0.5 * (last + end))
    return np.array(pts)


def _resolve(optimize, T, params, key, k, pts, h=None, scale_obj=-1e-5, **kw):
    """the case solved again with its parameter `key` of LP k (hour h of DA_LMPs) at each of pts -> PriceTakerResult of len(pts)"""
    M = len(pts)
    p = dict(params)
    lmp = np.repeat(np.asarray(params["DA_LMPs"], float)[[k]], M, axis=0)
    if h is not None:
        lmp[:, h] = pts
    p["DA_LMPs"] = lmp
    p["wind_resource"] = np.repeat(np.asarray(params["wind_resource"], float)[[k]], M, axis=0)        # one series per scenario
    for q in ("wind_mw", "batt_mw", "pem_mw", "h2_price_per_kg"):
        if q in params:
            p[q] = np.repeat(np.broadcast_to(np.asarray(params[q], float), (len(params["DA_LMPs"]),))[[k]], M)
    if key != "lmp":
        p[key] = pts
    return optimize(T, p, **kw)


def _check_renewables(optimize, params, T, names):
    res = optimize(T, params, want_curves={n: math.inf for n in names})
    assert (res.status == S.OPTIMAL).all() and set(res.curves) == set(names)
    checked = 0
    for name in names:
        cv = res.curves[name]
        assert (cv.status == S.OPTIMAL).all(), (name, cv.status)
        for k in range(LPS):
            for h in (HOURS if name == "lmp" else (None,)):
                idx = (k, h) if h is not None else (k,)
                pts = _points(cv, idx, math.inf)
                again = _resolve(optimize, T, params, name, k, pts, h, want_ranges=True, want_sensitivities=name == "lmp")
                assert (again.status == S.OPTIMAL).all()
                want = -1e-5 * cv.value(pts[None] if h is None else pts[None, None])[idx]          # NPV -> the objective
                err = np.abs(again.obj - want) / np.maximum(1.0, np.abs(again.obj))
                assert err.max() <= PRED_REL, (name, k, h, pts, again.obj, want)
                if name == "lmp":            # the slope: d NPV / d LMP of the hour = the vertex's sold energy in NPV units
                    e = np.clip(np.searchsorted(cv.at[idx][:cv.count[idx]], pts, side="right") - 1, 0, None)
                    slope = cv.slope[idx][e]
                    sold = again.marginal_npv["lmp"][:, h]
                    assert np.allclose(slope, sold, rtol=1e-9, atol=1e-9 * np.abs(sold).max()), (k, h, slope, sold)
                checked += len(pts)
    return res, checked


def test_wind_battery_want_curves():
    T, N = 24, 3
    lmp, cf, W, P = SC.c2(N, seed=11)
    params = {"wind_mw": W, "batt_mw": P, "wind_resource": np.tile(cf, (N, 1)), "DA_LMPs": lmp}
    res, checked = _check_renewables(PT.wind_battery_optimize, params, T, ("lmp", "wind_mw", "batt_mw"))
    assert res.curves["lmp"].at.shape[:2] == (N, T) and res.curves["batt_mw"].at.shape[0] == N
    assert (res.curves["batt_mw"].at[:, 0] == P).all()
    print("wind_battery: re-solved", checked, "points")
    with pytest.raises(ValueError):
        PT.wind_battery_optimize(T, params, want_curves={"batt_mw": P - 1.0})
    with pytest.raises(ValueError):
        PT.wind_battery_optimize(T, params, want_curves={"size": 1.0})


def test_wind_battery_pem_want_curves():
    T, N = 24, 3
    lmp, cf, W, _ = SC.c2(N, seed=5)
    params = {"wind_mw": W, "batt_mw": 0.0, "pem_mw": 200.0, "h2_price_per_kg": 2.5, "design_opt": False, "extant_wind": True,
              "wind_resource": np.tile(cf, (N, 1)), "DA_LMPs": lmp}
    res, checked = _check_renewables(PT.wind_battery_pem_optimize, params, T, ("lmp", "pem_mw", "h2_price_per_kg", "batt_mw"))
    print("wind_battery_pem: re-solved", checked, "points")


def test_nuclear_want_curves():
    T = 24
    s = R.nuclear(T, N=4)
    res = PT.nuclear_dispatch_optimize(T, s.cparams, want_curves={"lmp": math.inf})
    cv = res.curves["lmp"]
    assert (res.status == S.OPTIMAL).all() and cv.at.shape[:2] == (4, T) and (cv.status == S.OPTIMAL).all()
    for k in range(LPS):
        for h in HOURS:
            pts = _points(cv, (k, h), math.inf)
            moved = np.repeat(res.lmp[[k]], len(pts), axis=0)
            moved[:, h] = pts
            again = PT.nuclear_dispatch_optimize(T, moved, want_ranges=True, want_sensitivities=True)
            want = cv.value(pts[None, None])[k, h]
            err = np.abs(again.obj - want) / np.maximum(1.0, np.abs(again.obj))
            assert err.max() <= PRED_REL, (k, h, pts, again.obj, want)
            e = np.clip(np.searchsorted(cv.at[k, h][:cv.count[k, h]], pts, side="right") - 1, 0, None)
            sold = again.marginal_obj["lmp"][:, h]
            assert np.allclose(cv.slope[k, h][e], sold, rtol=1e-9, atol=1e-9 * max(1.0, np.abs(sold).max())), (k, h)
