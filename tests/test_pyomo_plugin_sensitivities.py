"""The Pyomo plugin's sensitivities (GPU): ``model.rc`` written back when the model declares an IMPORT ``rc`` Suffix, and
``res.batch["d_params"]`` with ``options={"sensitivities": True}``, on the reference-shaped wind + battery model of
tests/test_pyomo_plugin.py (tests/pyomo_stub where Pyomo is absent)."""
import numpy as np
import pytest

import exact_lp as E
from dispatches_b200.lp_template import model_reduced_costs
from oracle import highs as H, lp_models as L
from test_pyomo_plugin import PP, build_wind_battery, pyo

from dispatches_b200 import scenarios as SC

pytestmark = pytest.mark.gpu


def test_rc_suffix_agrees_with_the_exact_optimum_where_the_reduced_cost_is_unique():
    T = 24
    lmp, cf, W, P = SC.c2(64)
    m = build_wind_battery(T, lmp[0], cf, W, P)
    m.rc = pyo.Suffix(direction=pyo.Suffix.IMPORT)
    res = pyo.SolverFactory("b200ipm").solve(m)
    assert res.solver.termination_condition == pyo.TerminationCondition.optimal
    # the walked LP's exact optimum (HiGHS basis, verified in rational arithmetic) and its model-space reduced costs
    t, vars_, cons, p0 = PP.walk_model(m)
    e = E.exact_optimum(t, np.zeros(t.Pc), np.zeros(t.Pr))
    want = model_reduced_costs(t, e.y[None])[0]
    got = np.array([m.rc[v] for v in vars_])
    scale = np.abs(want).max()
    rec = t.meta["recover"]
    pos = {nm: q for q, nm in enumerate(t.col_names)}
    unique = np.zeros(len(vars_), bool)
    for j in range(len(vars_)):
        if rec["kind"][j] in (1, 2, 4):
            q = pos[rec["names"][rec["col"][j]]]
            unique[j] = e.unique_y or e.inside[q]          # rc unique: every optimal y, or a column strictly inside its bounds
    assert unique.sum() > 2 * T
    err = np.abs(got - want)[unique].max()
    assert err <= 1e-6 * scale, (err, scale)


def test_d_params_against_a_central_difference_in_the_windiest_hour():
    T = 24
    lmp, cf, W, P = SC.c2(8)
    m = build_wind_battery(T, lmp[0], cf, W, P)
    res = pyo.SolverFactory("b200ipm").solve(m, batch_params={m.blocks[t].lmp_signal: lmp[:, t] for t in range(T)},
                                             options={"sensitivities": True})
    d = res.batch["d_params"]
    assert d.shape == (8, T) and (res.batch["status"] == 0).all()
    t0 = int(np.argmax(cf))                        # the windiest hour: energy is sold there, the derivative is -1e-5 x its revenue rate
    eps = 1e-2
    for k in range(3):
        up, dn = lmp[k].copy(), lmp[k].copy()
        up[t0] += eps; dn[t0] -= eps
        fd = (H.solve(L.wind_battery_raw(up, cf, W, P))[0] - H.solve(L.wind_battery_raw(dn, cf, W, P))[0]) / (2 * eps)
        assert d[k, t0] == pytest.approx(fd, rel=1e-4, abs=1e-9), (k, d[k, t0], fd)
        assert d[k, t0] < 0
