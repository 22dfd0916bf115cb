"""The crossover through the user-facing paths (GPU): the Pyomo plugin's ``options={"crossover": True}`` on the reference-shaped
wind + battery model (tests/pyomo_stub where Pyomo is absent), and the double loop's ``solver={"crossover": True}`` against the
reference's known answers (tests/golden/double_loop_golden.json)."""
import numpy as np
import pytest

import exact_lp as E
from dispatches_b200 import double_loop as DLH, scenarios as SC, solver as S, templates as TP
from dispatches_b200.lp_template import model_duals, model_reduced_costs, model_values
from oracle import double_loop as DL, highs as H
from test_double_loop import CF, G, SIZES, _forecasts, _model
from test_pyomo_plugin import PP, build_wind_battery, pyo

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _template_vertex(t):
    """the walked template's vertex through the device API, the same kernels and options as the plugin"""
    sol = S.BatchLPSolver(t, native_setup=True)
    cp = torch.zeros((1, t.Pc), dtype=torch.float64, device="cuda")
    rp = torch.zeros((1, t.Pr), dtype=torch.float64, device="cuda") if t.Pr else None
    r = sol.solve(cp, rp, want_x=True, want_y=True)
    v = sol.crossover(cp, rp, r)
    return {k: getattr(v, k).cpu().numpy()[0] for k in ("obj", "x", "y", "col_status", "row_basic", "status")}


def test_plugin_loads_a_vertex_with_basis_duals():
    T = 24
    lmp, cf, W, P = SC.c2(64)
    m = build_wind_battery(T, lmp[0], cf, W, P)
    m.dual = pyo.Suffix(direction=pyo.Suffix.IMPORT)
    m.rc = pyo.Suffix(direction=pyo.Suffix.IMPORT)
    res = pyo.SolverFactory("b200ipm").solve(m, options={"crossover": True})
    assert res.solver.termination_condition == pyo.TerminationCondition.optimal
    assert (res.batch["crossover"]["status"] == 0).all()
    t, vars_, cons, p0 = PP.walk_model(m)
    v = _template_vertex(t)
    assert v["status"] == 0
    # the template's basis is an exact optimum, and the model's values, duals and reduced costs are that vertex's
    e = E.exact_optimum(t, np.zeros(t.Pc), np.zeros(t.Pr), basis=(v["col_status"].astype(np.int8), v["row_basic"].astype(bool)))
    assert np.abs(v["x"] - e.x).max() <= 1e-9 * max(1.0, np.abs(e.x).max())
    assert np.array_equal(res.batch["crossover"]["col_status"][0], v["col_status"])
    xm = model_values(t, v["x"][None], p0[None] if p0.size else np.zeros((1, 0)))[0]
    got = np.array([vv.value for vv in vars_])
    assert np.abs(got - xm).max() <= 1e-12 * max(1.0, np.abs(xm).max())
    ym = model_duals(t, v["y"][None])[0]
    assert np.abs(np.array([m.dual[c] for c in cons]) - ym).max() <= 1e-12 * max(1.0, np.abs(ym).max())
    rcm = model_reduced_costs(t, v["y"][None], p0[None] if p0.size else np.zeros((1, 0)))[0]
    assert np.abs(np.array([m.rc[vv] for vv in vars_]) - rcm).max() <= 1e-12 * max(1.0, np.abs(rcm).max())
    assert res.problem.upper_bound == pytest.approx(t.meta["sense"] * e.obj, rel=1e-9, abs=1e-9)


def test_plugin_batched_solve_returns_vertices():
    T = 24
    lmp, cf, W, P = SC.c2(8)
    m = build_wind_battery(T, lmp[0], cf, W, P)
    res = pyo.SolverFactory("b200ipm").solve(m, batch_params={m.blocks[t].lmp_signal: lmp[:, t] for t in range(T)},
                                             options={"crossover": True})
    xo = res.batch["crossover"]
    assert (res.batch["status"] == 0).all() and (xo["status"] == 0).all()
    assert xo["col_status"].shape[0] == 8 and set(np.unique(xo["col_status"])) <= {0, 1, 2}
    assert not hasattr(res.solver, "message") or res.solver.message is None
    t, vars_, cons, p0 = PP.walk_model(m, batch_params=[m.blocks[h].lmp_signal for h in range(T)])
    for k in range(8):
        basis = (xo["col_status"][k].astype(np.int8), xo["row_basic"][k].astype(bool))
        e = E.exact_optimum(t, lmp[k], lmp[k] if t.Pr else None, basis=basis)
        assert res.batch["obj"][k] == pytest.approx(t.meta["sense"] * e.obj, rel=1e-9, abs=1e-9)


def test_double_loop_tracker_known_answer_with_crossover():
    g = G["tracker"]
    tr = DLH.Tracker(tracking_model_object=_model(), tracking_horizon=4, n_tracking_hour=1, solver={"crossover": True})
    tr.track_market_dispatch(market_dispatch=g["market_dispatch"], date="2020-01-02", hour="00:00")
    wind = (tr.fs.sol["grid"] + tr.fs.sol["batt_in"])[0]
    assert wind == pytest.approx(g["expected_wind_power"], rel=g["rel"])
    assert tr.power_output[0] == pytest.approx(g["market_dispatch"], abs=g["abs_power"])
    assert tr.fs.sol["batt_in"][0] == pytest.approx(np.array(g["expected_wind_power"]) - 1e3 * np.array(g["market_dispatch"]), rel=g["rel"])


def test_double_loop_bids_with_crossover():
    bc = DLH.Backcaster({"Carter": G["da_309"]}, {"Carter": G["rt_309"]})
    ss = DLH.SelfScheduler(bidding_model_object=_model(), day_ahead_horizon=48, real_time_horizon=4, n_scenario=1, forecaster=bc,
                           solver={"crossover": True})
    bids = ss.compute_day_ahead_bids(date="2020-01-02")
    energies = np.array([b["309_WIND_1"]["p_max"] for b in bids.values()])
    known = np.array(G["self_schedule"]["known_solution"])
    ref_obj, _ = H.solve(DL.bidder_raw(*_forecasts(), CF, **SIZES))
    assert -ss.day_ahead_model.objective[0] == pytest.approx(ref_obj, rel=1e-8)
    # where the optimum is unique the vertex is CBC's; where da == rt or at hour 5 (two equally priced charging hours) the LP has other
    # optimal vertices, and CBC's is one of them
    da_f, rt_f = _forecasts()
    uniq = np.abs(da_f - rt_f) > 1e-9; uniq[5] = False
    assert np.allclose(energies[uniq], known[uniq], rtol=G["self_schedule"]["reltol"], atol=2e-3)
    print("hours where the vertex's bid differs from CBC's:", np.flatnonzero(~np.isclose(energies, known, rtol=1e-6, atol=2e-3)))


def test_48h_self_schedule_with_equal_prices_is_a_verified_vertex():
    """48-h day-ahead bidder LPs with DA == RT prices (every day-ahead quantity has zero cost: a whole face of optima)"""
    T, N = 48, 8
    rng = np.random.default_rng(4)
    p = SC.pool()
    idx = rng.integers(0, len(p["dalmp_303"]) - T, N)[:, None] + np.arange(T)[None, :]
    da = p["dalmp_303"][idx]
    rp = TP.wind_battery_operation_rparams(T, p["dacf_303"][idx], 200.0, 25.0, 100.0, rng.uniform(0, 90000, N), rng.uniform(0, 5000, N),
                                           None)
    cp = np.concatenate([da, da, np.full((N, 1), 1e3)], axis=1)
    t = TP.wind_battery_operation(T, "bidder_da")
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
    cpd, rpd = torch.as_tensor(cp, device="cuda"), torch.as_tensor(np.ascontiguousarray(rp), device="cuda")
    r = sol.solve(cpd, rpd, want_x=True, want_y=True)
    v = sol.crossover(cpd, rpd, r)
    st, cs, rb, x = (a.cpu().numpy() for a in (v.status, v.col_status, v.row_basic, v.x))
    assert (r.status.cpu().numpy() == 0).all() and (st == 0).all()
    for k in range(N):
        e = E.exact_optimum(t, cp[k], rp[k], basis=(cs[k].astype(np.int8), rb[k].astype(bool)))
        assert np.abs(x[k] - e.x).max() <= 1e-9 * max(1.0, np.abs(e.x).max())
