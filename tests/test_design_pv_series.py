"""PV + battery + hydrogen design optimisation with a PV and a reserve series per scenario (templates.solar_battery_hydrogen_design(T, None):
cf_t as per-problem matrix coefficients of the added-PV column): the per-problem template against the baked one and the raw oracle LP,
the numpy mirror of the dense kernel on per-problem instantiations (LPTemplate.matrix), and the argument checks of
pv_battery_hydrogen_design_optimize.  CPU only."""
import json
from pathlib import Path

import numpy as np
import pytest
from scipy.optimize import linprog

from dispatches_b200 import pricetaker as PT, templates as TP
from oracle import highs as H, ipm_dense_numpy as ID, lp_models as L

GOLD = json.load(open(Path(__file__).parent / "golden" / "solar_golden.json"))
LMP = np.array(GOLD["lmp_24"])
PAR = dict(pv_mw=0.0, turb_mw=0.0)


def dyadic_cfs(T, seed, zero_hours=False):
    """capacity factors on the 1/64 grid (strictly positive unless zero_hours): -(0.5 + (cf - 0.5)) is -cf exactly"""
    rng = np.random.default_rng(seed)
    d = np.tile(L.solar_default_series()["pv_cfs"], T // 24)
    cf = np.clip(np.round(d * rng.uniform(0.6, 1.0, T) * 64), 1, 64) / 64
    if zero_hours:
        cf[rng.choice(T, T // 4, replace=False)] = 0.0
    return cf


def solve_lp(A, c, b, u, k):
    r = linprog(c, A_eq=A, b_eq=b, bounds=[(0, None if not np.isfinite(v) else v) for v in u], method="highs-ds")
    assert r.status == 0, r.message
    return r.fun + k, r.x


@pytest.mark.parametrize("T,pv_mw", [(24, 0.0), (48, 0.0), (24, 50.0)])
def test_per_problem_template_is_the_baked_template(T, pv_mw):
    """at the same dyadic PV series and reserve: the same pattern, row and column order, and A, c, u and the objective constant bit for
    bit (b too when pv_mw = 0; otherwise cf_t * pv_mw is formed as 0.5 pv_mw + (cf_t - 0.5) pv_mw, equal to rounding)"""
    cf = dyadic_cfs(T, T)
    reserve = np.linspace(60.0, 110.0, T)
    lmp = np.tile(LMP, T // 24)
    load = np.linspace(80.0, 120.0, T)
    tb = TP.solar_battery_hydrogen_design(T, cf, reserve_mw=reserve, pv_mw=pv_mw)
    tp = TP.solar_battery_hydrogen_design(T, None, pv_mw=pv_mw)
    assert tp.amap is not None and len(tp.amap[0]) == 2 * T and tp.Pr == 3 * T and tp.w > 32
    assert tb.col_names == tp.col_names and tb.row_names == tp.row_names
    rp = TP.solar_design_rparams(T, load, cf, reserve)[0]
    Ab, Ap = tb.A.tocsr(), tp.matrix(rp).tocsr()
    Ab.sort_indices(); Ap.sort_indices()
    assert np.array_equal(Ab.indptr, Ap.indptr) and np.array_equal(Ab.indices, Ap.indices) and np.array_equal(Ab.data, Ap.data)
    cb, bb, ub, kb = tb.instantiate(lmp, load * 1e3)
    cp, bp, up, kp = tp.instantiate(lmp, rp)
    assert np.array_equal(cb, cp) and np.array_equal(ub, up) and kb == kp
    if pv_mw == 0.0:
        assert np.array_equal(bb, bp)
    else:
        assert np.abs(bb - bp).max() <= 1e-12 * np.abs(bb).max()


def test_zero_hours_keep_the_entry_in_the_pattern():
    T = 24
    tp = TP.solar_battery_hydrogen_design(T, None)
    va = tp.column("pv_add_system_capacity")
    rows = set(tp.amap[0][tp.amap[1] == va])
    names = {tp.row_names[i] for i in rows}
    assert names == {f"pv_max[{t}]" for t in range(T)} | {f"min_reserve[{t}]" for t in range(T)}
    assert all(tp.A[i, va] == -TP.PV_CF_NOMINAL for i in rows)          # stored whatever the series: the kernels' pattern
    A = tp.matrix(TP.solar_design_rparams(T, np.full(T, 100.0), np.zeros(T), np.full(T, 100.0))[0]).tocsr()
    assert all(A[i, va] == 0.0 for i in rows)


def _cases():
    """(name, lmp, load, cfs, reserve): the reference's case, perturbed PV series with zero hours and one all-zero series, and a
    perturbed reserve series"""
    d = L.solar_default_series()
    rng = np.random.default_rng(7)
    out = [("reference", LMP, d["load_mw"], d["pv_cfs"], d["reserve_mw"])]
    for k in range(2):
        cf = d["pv_cfs"] * rng.uniform(0.5, 1.0, 24)
        cf[rng.choice(24, 5, replace=False)] = 0.0
        out.append((f"pv_zero_hours{k}", LMP * rng.lognormal(0, 0.3, 24), d["load_mw"] * rng.uniform(0.7, 1.2, 24), cf, d["reserve_mw"]))
    out.append(("pv_all_zero", LMP * rng.lognormal(0, 0.3, 24), d["load_mw"], np.zeros(24), d["reserve_mw"]))
    out.append(("reserve", LMP, d["load_mw"] * rng.uniform(0.7, 1.2, 24), d["pv_cfs"], 100.0 * rng.uniform(0.4, 1.0, 24)))
    return out


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_per_problem_template_matches_the_raw_oracle(case):
    name, lmp, load, cfs, reserve = case
    tp = TP.solar_battery_hydrogen_design(24, None, **PAR)
    rp = TP.solar_design_rparams(24, load, cfs, reserve)[0]
    c, b, u, k = tp.instantiate(lmp, rp)
    a, x = solve_lp(tp.matrix(rp), c, b, u, k)
    ref = H.solve(L.solar_battery_hydrogen_raw(lmp, True, PAR, pv_cfs=cfs, load_mw=load, reserve_mw=reserve))[0]
    assert a == pytest.approx(ref, rel=1e-10, abs=1e-8)
    if name == "reference":
        assert -a * 1e3 == pytest.approx(GOLD["test_solar_batt_hydrogen_optimize"]["expect"]["NPV"]["value"], rel=1e-8)


def test_dense_mirror_on_per_problem_instantiations():
    """the dense kernel's algebra (oracle/ipm_dense_numpy.py) on each LP's own matrix: OPTIMAL, within 1e-8 of HiGHS"""
    tp = TP.solar_battery_hydrogen_design(24, None, **PAR)
    for name, lmp, load, cfs, reserve in CASES:
        rp = TP.solar_design_rparams(24, load, cfs, reserve)[0]
        c, b, u, k = tp.instantiate(lmp, rp)
        r = ID.solve_batch(tp.matrix(rp), b[None], c[None], u[None], rho=tp.meta.get("reg_primal", 1e-8))
        ref = H.solve(L.solar_battery_hydrogen_raw(lmp, True, PAR, pv_cfs=cfs, load_mw=load, reserve_mw=reserve))[0]
        assert r["status"][0] == ID.OPTIMAL, name
        assert abs(r["obj"][0] + k - ref) / abs(ref) < 1e-8, name


def _params(T=24, **over):
    d = L.solar_default_series()
    p = dict(pv_mw=0.0, turb_mw=0.0, LMP=np.tile(LMP, (3, 1)), load=d["load_mw"], reserve=d["reserve_mw"], pv_resource=d["pv_cfs"])
    p.update(over)
    return p


@pytest.mark.parametrize("over,match", [
    (dict(pv_resource=np.full((3, 23), 0.5)), "pv_resource must be"),
    (dict(pv_resource=np.full((3, 24, 1), 0.5)), "pv_resource must be"),
    (dict(reserve=np.full((2, 2, 24), 100.0)), "reserve must be"),
    (dict(pv_resource=np.full((3, 24), -0.1)), "finite and >= 0"),
    (dict(pv_resource=np.r_[np.full(23, 0.5), np.nan]), "finite and >= 0"),
    (dict(pv_resource=np.r_[np.full(23, 0.5), np.inf]), "finite and >= 0"),
    (dict(reserve=np.r_[np.full(23, 100.0), np.nan]), "reserves finite"),
    (dict(pv_resource=np.full((2, 24), 0.5)), "one series or one per scenario"),
    (dict(reserve=np.full((4, 24), 100.0)), "one series or one per scenario"),
])
def test_design_optimize_argument_checks(over, match):
    with pytest.raises(ValueError, match=match):
        PT.pv_battery_hydrogen_design_optimize(24, _params(**over))


def test_design_rparams_layout():
    T = 24
    cf = np.linspace(0, 1, T); rs = np.arange(T, dtype=float); ld = np.full(T, 90.0)
    rp = TP.solar_design_rparams(T, ld, cf, rs)
    assert rp.shape == (1, 3 * T)
    assert np.array_equal(rp[0, :T], ld * 1e3) and np.array_equal(rp[0, T:2 * T], cf - TP.PV_CF_NOMINAL)
    assert rp[0, 2 * T] == rs[0] * 1e3 and np.array_equal(rp[0, 2 * T + 1:], rs[:-1] * 1e3)   # hour t asks the reserve of hour t - 1
