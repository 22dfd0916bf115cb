"""Host-side mirror of the reference's price-taker entry points, batched over LMP scenarios.

Same names and argument meaning as the reference functions; the only extension is that ``DA_LMPs`` may be a
2-D array [N, >=T] (one row per price scenario) and sizes may be arrays [N] (one entry per design point):

  wind_battery_optimize(n_time_points, input_params, verbose)     wind_battery_LMP.py:172-269
  wind_battery_pem_optimize(time_points, input_params, verbose)    wind_battery_PEM_LMP.py:180-298
  record_results(res)                                              wind_battery_LMP.py:272-325
  nuclear_dispatch_optimize(n_time_points, lmps, ...)              nuclear_flowsheet_multiperiod_class.py:72-155
  pv_battery_hydrogen_optimize(n_time_points, input_params, ...)   solar_battery_hydrogen.py:375-606 (design_opt=False)
  pv_battery_hydrogen_design_optimize(n_time_points, input_params, ...)   the same with design_opt=True (dense kernel)

Where the reference builds a Pyomo MultiPeriodModel and calls SolverFactory("cbc").solve(m) once per signal,
these build (and cache) one LPTemplate per (flowsheet, T) and hand the whole batch to the CUDA solver.
``design_opt=True`` (battery size; with ``extant_wind=False`` also the wind size, for one capacity-factor series per call)
and ``design_opt="PEM"`` run on the same path: capacity columns are kept per period with link equalities (banded).
"""
from __future__ import annotations

import dataclasses

import numpy as np

from . import templates as TP
from .solver import KERNEL_DENSE, BatchLPSolver, OPTIMAL, STATUS_NAMES

_SOLVERS = {}


def get_solver(kind, T, **kw) -> BatchLPSolver:
    key = (kind, T, tuple(sorted(kw.items())))
    if key not in _SOLVERS:
        builder = dict(wind_battery=TP.wind_battery, wind_battery_design=TP.wind_battery_design,
                       wind_battery_pem=TP.wind_battery_pem, nuclear=TP.nuclear,
                       fossil_surrogate=TP.fossil_surrogate)[kind]
        _SOLVERS[key] = BatchLPSolver(builder(T, **kw))
    return _SOLVERS[key]


def _capacity_factors(input_params, T):
    wr = input_params["wind_resource"]
    if isinstance(wr, dict):       # the reference's {t: {'wind_resource_config': {'capacity_factor': [cf]}}}
        return np.array([wr[t]["wind_resource_config"]["capacity_factor"][0] for t in range(T)], float)
    wr = np.asarray(wr, float)
    return wr[..., :T]


@dataclasses.dataclass
class PriceTakerResult:
    kind: str
    T: int
    lmp: np.ndarray                 # [N,T] $/MWh
    obj: np.ndarray                 # [N]   the reference Objective value (-NPV*1e-5 for the renewables cases)
    status: np.ndarray
    iters: np.ndarray
    x: np.ndarray | None            # [N,n] model-space values of the template columns
    col_names: list
    sizes: dict

    @property
    def NPV(self):
        return -self.obj * 1e5

    @property
    def termination_condition(self):
        return [STATUS_NAMES[int(s)] for s in self.status]

    def var(self, name, t=None):
        """Values [N] of a reference Var, e.g. var("battery.state_of_charge[0]", t=3)."""
        full = name if t is None else f"blk[{t}].fs.{name}"
        if full in self.col_names:
            return self.x[:, self.col_names.index(full)]
        if self.kind.startswith("wind_battery") and full == f"blk[{self.T - 1}].fs.battery.state_of_charge[0]":
            return np.zeros(self.x.shape[0])       # presolved constant (periodic constraint)
        raise KeyError(full)

    def series(self, name):
        """[N,T] time series of a per-period Var."""
        return np.stack([self.var(name, t) for t in range(self.T)], axis=1)

    # quantities the reference exposes as model Expressions (wind_battery_LMP.py:252-263)
    @property
    def annual_elec_revenue(self):
        ann = 52.0 / (self.T / 168.0)
        out = self.series("splitter.grid_elec[0]")
        try:
            out = out + self.series("battery.elec_out[0]")
        except KeyError:
            pass
        return (self.lmp * 1e-3 * out).sum(1) * ann

    @property
    def annual_revenue(self):
        ann = 52.0 / (self.T / 168.0)
        fixed = self.sizes["wind_kw"] * TP.WIND_OP_COST / 8760.0 + self.sizes["batt_kw"] * TP.BATT_OP_COST / 8760.0
        rev = self.annual_elec_revenue
        if "pem_kw" in self.sizes:
            fixed = fixed + self.sizes["pem_kw"] * TP.PEM_OP_COST / 8760.0
            rev = rev + self.annual_rev_h2
        return rev - fixed * self.T * ann

    @property
    def annual_rev_h2(self):
        ann = 52.0 / (self.T / 168.0)
        pe = self.series("pem.electricity[0]")
        return pe.sum(1) * TP.PEM_ELEC_TO_MOL / TP.H2_MOLS_PER_KG * 3600.0 * self.sizes["h2_price"] * ann


def _lmps(input_params, T):
    lmp = np.asarray(input_params["DA_LMPs"], float)
    lmp = np.atleast_2d(lmp)[:, :T]
    if lmp.shape[1] != T:
        raise ValueError(f"DA_LMPs must provide {T} values per scenario")
    return np.ascontiguousarray(lmp)


def wind_battery_optimize(n_time_points, input_params, verbose=False, want_solution=True):
    T = int(n_time_points)
    design = bool(input_params.get("design_opt", False))
    lmp = _lmps(input_params, T)
    cf = _capacity_factors(input_params, T)
    if design and not input_params.get("extant_wind", True):
        return _wind_battery_free_wind(T, lmp, cf, input_params, verbose)
    sol = get_solver("wind_battery_design" if design else "wind_battery", T,
                     extant_wind=bool(input_params.get("extant_wind", True)))
    want_solution = want_solution or design          # the optimal battery size is read from the solution
    rp = TP.wind_battery_rparams(T, cf, input_params["wind_mw"], input_params["batt_mw"])
    if rp.shape[0] == 1:
        rp = rp[0]
    elif rp.shape[0] != lmp.shape[0]:
        raise ValueError("sizes / capacity factors must be scalar or match the number of LMP scenarios")
    r = sol.solve_host(lmp, rp, want_x=want_solution)
    if verbose:
        print(f"b200ipm: {lmp.shape[0]} LPs, iterations mean {r.iters.mean():.1f} max {r.iters.max()}, "
              f"non-optimal {(r.status != OPTIMAL).sum()}")
    N = lmp.shape[0]
    sizes = dict(wind_kw=np.broadcast_to(np.asarray(input_params["wind_mw"], float) * 1e3, (N,)),
                 batt_kw=np.broadcast_to(np.asarray(input_params["batt_mw"], float) * 1e3, (N,)))
    xm = sol.to_model_space(r.x) if want_solution else None
    if design:                                        # optimised size: value(m.battery_system_capacity)
        sizes["batt_kw"] = xm[:, sol.t.col_names.index("blk[0].fs.battery.nameplate_power")].copy()
    return PriceTakerResult("wind_battery", T, lmp, r.obj, r.status, r.iters, xm, sol.t.col_names, sizes)


def _wind_battery_free_wind(T, lmp, cf, input_params, verbose):
    """design_opt=True, extant_wind=False: battery and wind size are decisions (wind_battery_LMP.py:209-219).  cf_t
    multiplies the wind-capacity column: with ONE series it is baked into the template (batch over LMP scenarios); with a
    series per scenario the cf_t become per-problem matrix coefficients of the band kernel."""
    cf = np.asarray(cf, float)
    ub = float(input_params.get("wind_mw_ub", 10000.0))
    rp = None
    if cf.ndim != 1 and not np.all(cf == cf[:1]):
        # a capacity-factor series per batch member: cf_t multiplies the wind-capacity column, i.e. it is a coefficient of the
        # constraint matrix -> per-problem matrix coefficients (templates.wind_battery_design_free_wind(cf=None))
        if cf.shape[0] != lmp.shape[0]:
            raise ValueError("wind_resource must be one series or one per LMP scenario")
        key = ("wind_battery_design_free_wind_cfbatched", T, ub)
        if key not in _SOLVERS:
            _SOLVERS[key] = BatchLPSolver(TP.wind_battery_design_free_wind(T, None, ub))
        rp = np.ascontiguousarray(cf - TP.CF_NOMINAL)
    else:
        if cf.ndim != 1:
            cf = cf[0]
        key = ("wind_battery_design_free_wind", T, cf.tobytes(), ub)
        if key not in _SOLVERS:
            _SOLVERS[key] = BatchLPSolver(TP.wind_battery_design_free_wind(T, cf, ub))
    sol = _SOLVERS[key]
    r = sol.solve_host(lmp, rp, want_x=True)
    if verbose:
        print(f"b200ipm: {lmp.shape[0]} LPs, iterations mean {r.iters.mean():.1f} max {r.iters.max()}, "
              f"non-optimal {(r.status != OPTIMAL).sum()}")
    xm = sol.to_model_space(r.x)
    names = sol.t.col_names
    sizes = dict(wind_kw=xm[:, names.index("blk[0].fs.windpower.system_capacity")].copy(),      # value(m.wind_system_capacity)
                 batt_kw=xm[:, names.index("blk[0].fs.battery.nameplate_power")].copy())         # value(m.battery_system_capacity)
    return PriceTakerResult("wind_battery", T, lmp, r.obj, r.status, r.iters, xm, names, sizes)


def wind_battery_pem_optimize(time_points, input_params, verbose=False, want_solution=True):
    mode = input_params.get("design_opt", False)
    if mode not in (False, "PEM") or (mode == "PEM" and not input_params.get("extant_wind", True)):
        raise NotImplementedError("only design_opt False and \"PEM\" (extant wind) are on the batched GPU path")
    pem_design = mode == "PEM"
    T = int(time_points)
    lmp = _lmps(input_params, T)
    N = lmp.shape[0]
    cf = _capacity_factors(input_params, T)
    batt = np.zeros(1) if pem_design else np.asarray(input_params["batt_mw"], float)   # "PEM" fixes the battery at 0 (:228)
    with_batt = bool(np.any(batt > 0))
    want_solution = want_solution or pem_design
    sol = get_solver("wind_battery_pem", T, with_battery=with_batt, extant_wind=bool(input_params.get("extant_wind", True)),
                     pem_design=pem_design)
    rp = TP.wind_battery_rparams(T, cf, input_params["wind_mw"], batt, pem_mw=input_params["pem_mw"])
    if rp.shape[0] == 1:
        rp = rp[0]
    elif rp.shape[0] != N:
        raise ValueError("sizes / capacity factors must be scalar or match the number of LMP scenarios")
    h2 = np.broadcast_to(np.asarray(input_params["h2_price_per_kg"], float), (N,))
    cp = np.ascontiguousarray(np.concatenate([lmp, h2[:, None]], axis=1))
    r = sol.solve_host(cp, rp, want_x=want_solution)
    sizes = dict(wind_kw=np.broadcast_to(np.asarray(input_params["wind_mw"], float) * 1e3, (N,)),
                 batt_kw=np.broadcast_to(batt * 1e3, (N,)),
                 pem_kw=np.broadcast_to(np.asarray(input_params["pem_mw"], float) * 1e3, (N,)), h2_price=h2)
    xm = sol.to_model_space(r.x) if want_solution else None
    if pem_design:                                    # optimised size: value(m.pem_system_capacity)
        sizes["pem_kw"] = xm[:, sol.t.col_names.index("pem_system_capacity[0]")].copy()
    return PriceTakerResult("wind_battery_pem", T, lmp, r.obj, r.status, r.iters, xm, sol.t.col_names, sizes)


def nuclear_dispatch_optimize(n_time_points, lmps, want_solution=False, **flowsheet_options):
    T = int(n_time_points)
    lmp = np.ascontiguousarray(np.atleast_2d(np.asarray(lmps, float))[:, :T])
    sol = get_solver("nuclear", T, **flowsheet_options)
    r = sol.solve_host(lmp, None, want_x=want_solution)
    return PriceTakerResult("nuclear", T, lmp, r.obj, r.status, r.iters,
                            sol.to_model_space(r.x) if want_solution else None, sol.t.col_names, {})


_SOLAR_COST_KEYS = ("pv_cap_cost", "pv_op_cost", "batt_cap_cost_kw", "batt_cap_cost_kwh", "pem_cap_cost", "pem_op_cost", "pem_var_cost",
                    "tank_cap_cost_per_kg", "tank_op_cost", "turbine_cap_cost", "turbine_op_cost", "turbine_var_cost", "h2_price_per_kg",
                    "turbine_min_mw", "turbine_ramp_mw_per_min", "h2_turb_conv")


def pv_battery_hydrogen_optimize(n_time_points, input_params, verbose=False, plot=False):
    """The reference's PV + battery + PEM + hydrogen tank + turbine load-following case (solar_battery_hydrogen.py:375-606) with
    ``design_opt=False``, batched: ``LMP`` [T] or [N, T], ``load`` / ``pv_resource`` [T] or [N, T].  Same ``input_params`` keys as
    ``re_h2_parameters`` (solar_battery_hydrogen_inputs.py:79-118).  Returns (design_res, df) like the reference: ``design_res`` with
    the reference's keys (scalars, or arrays [N] for a batch), ``df`` a dict of the operating series [N, T] under the
    reference's column names (one pandas frame per scenario is a ``pd.DataFrame({k: v[i] for k, v in df.items()})`` away).
    design_opt=True is refused here: its six size variables couple every period (not banded within the band kernel's limit);
    pv_battery_hydrogen_design_optimize solves it on the dense kernel."""
    if input_params.get("design_opt", False):
        raise NotImplementedError("pv_battery_hydrogen_optimize: design_opt=True is not on the band kernels' path "
                                  "(six dense size columns); use pv_battery_hydrogen_design_optimize (dense kernel)")
    T = int(n_time_points)
    for k in ("LMP", "pv_resource", "load", "reserve", "pv_mw", "tank_size", "turb_mw"):
        if k not in input_params:
            raise KeyError(f"pv_battery_hydrogen_optimize: input_params[{k!r}] is required")
    lmp = np.ascontiguousarray(np.atleast_2d(np.asarray(input_params["LMP"], float))[:, :T])
    pr = input_params["pv_resource"]
    if isinstance(pr, dict):       # the reference's {t: {'pv_resource_config': {'capacity_factor': cf}}}
        cfs = np.array([np.ravel(pr[t]["pv_resource_config"]["capacity_factor"])[0] for t in range(T)], float)
    else:
        cfs = np.asarray(pr, float)[..., :T]
    load = np.asarray(input_params["load"], float)[..., :T]
    for name, a in (("LMP", lmp), ("pv_resource", cfs), ("load", load), ("reserve", np.asarray(input_params["reserve"], float)[..., :T])):
        if a.shape[-1] != T or a.ndim > 2 or (name == "reserve" and a.ndim != 1):
            raise ValueError(f"pv_battery_hydrogen_optimize: {name} must provide {T} values per scenario (reserve: one series), got shape {a.shape}")
    if np.any(cfs < 0) or not np.all(np.isfinite(cfs)) or not np.all(np.isfinite(load)):
        raise ValueError("pv_battery_hydrogen_optimize: capacity factors must be finite and >= 0, loads finite")
    batt_mw = float(input_params.get("batt_mw", 0.0))
    batt_mwh = float(input_params["batt_mw"] * input_params["batt_hr"]) if "batt_hr" in input_params else float(input_params.get("batt_mwh", 0.0))
    par = {k: float(input_params[k]) for k in _SOLAR_COST_KEYS if k in input_params}
    kw = dict(batt_mw=batt_mw, batt_mwh=batt_mwh, pem_mw=float(input_params.get("pem_mw", 0.0)), tank_kg=float(input_params["tank_size"]),
              turb_mw=float(input_params["turb_mw"]), max_sales=float(input_params.get("max_sales", np.inf)),
              max_purchases=float(input_params.get("max_purchases", np.inf)))
    key = ("solar_battery_hydrogen", T, tuple(sorted(kw.items())), tuple(sorted(par.items())),
           np.asarray(input_params["reserve"], float)[:T].tobytes())
    if key not in _SOLVERS:
        _SOLVERS[key] = BatchLPSolver(TP.solar_battery_hydrogen(T, reserve_mw=np.asarray(input_params["reserve"], float)[:T], par=par, **kw))
    sol = _SOLVERS[key]
    t = sol.t
    rp = TP.solar_rparams(T, cfs, input_params["pv_mw"], load)
    N = max(lmp.shape[0], rp.shape[0])
    if lmp.shape[0] not in (1, N) or rp.shape[0] not in (1, N):
        raise ValueError("LMP, load and pv_resource must be one series or one per scenario")
    lmp = np.ascontiguousarray(np.broadcast_to(lmp, (N, T)))
    r = sol.solve_host(lmp, rp[0] if rp.shape[0] == 1 else rp, want_x=True)
    if verbose:
        print(f"b200ipm: {N} LPs, iterations mean {r.iters.mean():.1f} max {r.iters.max()}, non-optimal {(r.status != OPTIMAL).sum()}")
    xm = sol.to_model_space(r.x)
    names = {n: j for j, n in enumerate(t.col_names)}

    def ser(name, blk_level=False):
        cols = [names.get((f"blk[{k}]." if blk_level else f"blk[{k}].fs.") + name) for k in range(T)]
        return np.stack([xm[:, c] if c is not None else np.zeros(N) for c in cols], axis=1)
    P = dict(TP.SOLAR); P.update(par)
    sz = t.meta["sizes"]
    k_turb = t.meta["k_turb"]
    pv_kw = np.broadcast_to(np.asarray(input_params["pv_mw"], float) * 1e3, (N,))
    pv_gen, grid, pem = ser("pv.electricity[0]"), ser("splitter.grid_elec[0]"), ser("pem.electricity[0]")
    b_in, b_out, soc = ser("battery.elec_in[0]"), ser("battery.elec_out[0]"), ser("battery.state_of_charge[0]")
    to_turb, to_pipe, holdup = ser("h2_tank.outlet_to_turbine.flow_mol[0]"), ser("h2_tank.outlet_to_pipeline.flow_mol[0]"), ser("h2_tank.tank_holdup[0]")
    purchase, sales = ser("grid_purchase", True), ser("grid_sales", True)
    turb_elec = to_turb * k_turb
    n_weeks = T / 168.0
    h2_rev = P["h2_price_per_kg"] / TP.H2_MOLS_PER_KG * to_pipe * P["s_per_ts"]
    grid_cost = lmp * (purchase - sales) * 1e-3
    pem_var, turb_var = P["pem_var_cost"] * pem, P["turbine_var_cost"] * turb_elec
    fixed = pv_kw * P["pv_op_cost"] + sz["pem_kw"] * P["pem_op_cost"] + t.meta["tank_kg"] * P["tank_op_cost"] + sz["turb_kw"] * P["turbine_op_cost"]
    squeeze = (lambda a: float(a[0])) if N == 1 else (lambda a: a)
    design_res = {
        "pv_mw": squeeze(pv_kw * 1e-3), "batt_mw": sz["batt_kw"] * 1e-3, "batt_mwh": sz["batt_kwh"] * 1e-3,
        "batt_hr": sz["batt_kwh"] / sz["batt_kw"] if sz["batt_kw"] else 0, "pem_mw": sz["pem_kw"] * 1e-3,
        "tank_tonH2": t.meta["tank_kg"] * P["kg_to_tons"], "turb_mw": sz["turb_kw"] * 1e-3,
        "capital_cost": t.meta["capital_cost"], "capital_cost_pv": 0.0, "capital_cost_batt_kw": P["batt_cap_cost_kw"] * sz["batt_kw"],
        "capital_cost_batt_kwh": P["batt_cap_cost_kwh"] * sz["batt_kwh"], "capital_cost_pem": P["pem_cap_cost"] * sz["pem_kw"],
        "capital_cost_tank": P["tank_cap_cost_per_kg"] * t.meta["tank_kg"], "capital_cost_turb": 0.0,
        "annual_costs_fixed": squeeze(fixed), "fixed_cost_pv": squeeze(pv_kw * P["pv_op_cost"]), "fixed_cost_pem": sz["pem_kw"] * P["pem_op_cost"],
        "fixed_cost_tank": t.meta["tank_kg"] * P["tank_op_cost"], "fixed_cost_turb": sz["turb_kw"] * P["turbine_op_cost"],
        "annual_costs_variable": squeeze((pem_var + turb_var).sum(1)), "variable_cost_batt": 0.0,
        "variable_cost_pem": squeeze(pem_var.sum(1)), "variable_cost_turb": squeeze(turb_var.sum(1)),
        "annual_costs_NG": 0.0, "annual_costs_grid": squeeze(grid_cost.sum(1) * 52 / n_weeks),
        "annual_costs_total": squeeze((grid_cost + pem_var + turb_var).sum(1) * 52 / n_weeks),
        "annual_rev_h2": squeeze(h2_rev.sum(1) * 52 / n_weeks), "NPV": squeeze(-r.obj * 1e3), "CO2_lb": 0.0,
        "status": [STATUS_NAMES[int(v)] for v in r.status],
    }
    cf2 = np.broadcast_to(np.atleast_2d(cfs), (N, T))
    df = {
        "Total PV Generation [MW]": pv_gen * 1e-3, "Total Power Output [MW]": (grid + b_out + turb_elec) * 1e-3,
        "PV Power Output [MW]": grid * 1e-3, "PV Power to Battery [MW]": b_in * 1e-3,
        "State of Charge": soc / sz["batt_kwh"] if sz["batt_kwh"] else soc, "Battery Power Output [MW]": b_out * 1e-3,
        "PV Power to PEM [MW]": pem * 1e-3, "PEM H2 Output [kg]": pem * TP.PEM_ELEC_TO_MOL * P["s_per_ts"] / TP.H2_MOLS_PER_KG,
        "H2 Sales [kg]": to_pipe * P["s_per_ts"] / TP.H2_MOLS_PER_KG, "Turbine H2 Input [kg]": to_turb * P["s_per_ts"] / TP.H2_MOLS_PER_KG,
        "Turbine Power [MW]": turb_elec * 1e-3, "Purchased Power [MW]": purchase * 1e-3, "Sold Power [MW]": sales * 1e-3,
        "Tank Holdup [kg]": holdup / TP.H2_MOLS_PER_KG, "Excess PV [MW]": (pv_kw[:, None] * cf2 - pv_gen) * 1e-3,
        "Battery Reserve [MW]": ser("battery_reserve", True) * 1e-3, "PEM Reserve [MW]": pem * 1e-3,
        "Turbine Reserve [MW]": ser("turbine_reserve", True) * 1e-3, "Load [MW]": np.broadcast_to(np.atleast_2d(load), (N, T)),
        "Grid Income [$]": grid_cost, "H2 Revenue [$]": h2_rev, "Operating Cost [$]": pem_var + turb_var,
    }
    return design_res, df


def pv_battery_hydrogen_design_optimize(n_time_points, input_params, verbose=False):
    """The reference's PV + battery + PEM + hydrogen tank + turbine case with ``design_opt=True`` (solar_battery_hydrogen.py:375-606,
    size_constraints :205-236): the added PV, battery power / energy, PEM, tank and turbine sizes are decisions.  Batched over price and
    load series: ``LMP`` and ``load`` [T] or [N, T]; ``pv_resource`` and ``reserve`` one series (the PV capacity factors multiply the
    added-PV column, so they are part of the template).  Same ``input_params`` keys as ``re_h2_parameters``; ``pv_mw`` / ``turb_mw``
    are the existing PV and turbine sizes the design adds to.  Those six columns make A A' dense, so the LPs run on the dense kernel
    (m <= 1024: T <= 48).  Returns (design_res, df) like the reference, with the optimal sizes per scenario."""
    T = int(n_time_points)
    for k in ("LMP", "pv_resource", "load", "reserve"):
        if k not in input_params:
            raise KeyError(f"pv_battery_hydrogen_design_optimize: input_params[{k!r}] is required")
    lmp = np.ascontiguousarray(np.atleast_2d(np.asarray(input_params["LMP"], float))[:, :T])
    pr = input_params["pv_resource"]
    if isinstance(pr, dict):
        cfs = np.array([np.ravel(pr[t]["pv_resource_config"]["capacity_factor"])[0] for t in range(T)], float)
    else:
        cfs = np.asarray(pr, float)[..., :T]
    load = np.atleast_2d(np.asarray(input_params["load"], float))[:, :T]
    reserve = np.asarray(input_params["reserve"], float)[..., :T]
    for name, a in (("LMP", lmp), ("pv_resource", cfs), ("load", load), ("reserve", reserve)):
        if a.shape[-1] != T or (name in ("pv_resource", "reserve") and a.ndim != 1):
            raise ValueError(f"pv_battery_hydrogen_design_optimize: {name} must provide {T} values per scenario "
                             f"(pv_resource, reserve: one series), got shape {a.shape}")
    if np.any(cfs < 0) or not np.all(np.isfinite(cfs)) or not np.all(np.isfinite(load)):
        raise ValueError("pv_battery_hydrogen_design_optimize: capacity factors must be finite and >= 0, loads finite")
    N = max(lmp.shape[0], load.shape[0])
    if lmp.shape[0] not in (1, N) or load.shape[0] not in (1, N):
        raise ValueError("LMP and load must be one series or one per scenario")
    par = {k: float(input_params[k]) for k in _SOLAR_COST_KEYS if k in input_params}
    kw = dict(pv_mw=float(input_params.get("pv_mw", 0.0)), turb_mw=float(input_params.get("turb_mw", 0.0)),
              max_sales=float(input_params.get("max_sales", 1000.0)), max_purchases=float(input_params.get("max_purchases", 1000.0)))
    key = ("solar_battery_hydrogen_design", T, tuple(sorted(kw.items())), tuple(sorted(par.items())), cfs.tobytes(), reserve.tobytes())
    if key not in _SOLVERS:
        _SOLVERS[key] = BatchLPSolver(TP.solar_battery_hydrogen_design(T, cfs, reserve_mw=reserve, par=par, **kw), kernel=KERNEL_DENSE)
    sol = _SOLVERS[key]
    t = sol.t
    lmp = np.ascontiguousarray(np.broadcast_to(lmp, (N, T)))
    rp = np.ascontiguousarray(np.broadcast_to(load * 1e3, (N, T)))
    r = sol.solve_host(lmp, rp, want_x=True)
    if verbose:
        print(f"b200ipm (dense kernel): {N} LPs, iterations mean {r.iters.mean():.1f} max {r.iters.max()}, "
              f"non-optimal {(r.status != OPTIMAL).sum()}")
    xm = sol.to_model_space(r.x)
    names = {n: j for j, n in enumerate(t.col_names)}
    size = {nm: xm[:, names[nm]] for nm in TP.SOLAR_SIZE_COLUMNS}

    def ser(name, blk_level=False):
        return np.stack([xm[:, names[(f"blk[{k}]." if blk_level else f"blk[{k}].fs.") + name]] for k in range(T)], axis=1)
    P = dict(TP.SOLAR); P.update(par)
    k_turb = t.meta["k_turb"]
    pv_kw = kw["pv_mw"] * 1e3 + size["pv_add_system_capacity"]
    batt_kw, batt_kwh = size["battery_system_capacity"], size["battery_system_energy"]
    pem_kw, tank_kg, turb_kw = size["pem_system_capacity"], size["h2_tank_size"], size["turb_system_capacity"]
    grid, pem = ser("splitter.grid_elec[0]"), ser("pem.electricity[0]")
    b_in, b_out, soc = ser("battery.elec_in[0]"), ser("battery.elec_out[0]"), ser("battery.state_of_charge[0]")
    to_turb, to_pipe, holdup = ser("h2_tank.outlet_to_turbine.flow_mol[0]"), ser("h2_tank.outlet_to_pipeline.flow_mol[0]"), ser("h2_tank.tank_holdup[0]")
    purchase, sales = ser("grid_purchase", True), ser("grid_sales", True)
    turb_elec = to_turb * k_turb
    n_weeks = T / 168.0
    h2_rev = P["h2_price_per_kg"] / TP.H2_MOLS_PER_KG * to_pipe * P["s_per_ts"]
    grid_cost = lmp * (purchase - sales) * 1e-3
    pem_var, turb_var = P["pem_var_cost"] * pem, P["turbine_var_cost"] * turb_elec
    cap_pv, cap_kw, cap_kwh = P["pv_cap_cost"] * size["pv_add_system_capacity"], P["batt_cap_cost_kw"] * batt_kw, P["batt_cap_cost_kwh"] * batt_kwh
    cap_pem, cap_tank = P["pem_cap_cost"] * pem_kw, P["tank_cap_cost_per_kg"] * tank_kg
    cap_turb = P["turbine_cap_cost"] * (turb_kw - kw["turb_mw"] * 1e3)
    fixed = pv_kw * P["pv_op_cost"] + pem_kw * P["pem_op_cost"] + tank_kg * P["tank_op_cost"] + turb_kw * P["turbine_op_cost"]
    squeeze = (lambda a: float(np.ravel(a)[0])) if N == 1 else (lambda a: np.asarray(a))
    design_res = {
        "pv_mw": squeeze(pv_kw * 1e-3), "batt_mw": squeeze(batt_kw * 1e-3), "batt_mwh": squeeze(batt_kwh * 1e-3),
        "batt_hr": squeeze(np.where(batt_kw > 0, batt_kwh / np.where(batt_kw > 0, batt_kw, 1.0), 0.0)), "pem_mw": squeeze(pem_kw * 1e-3),
        "tank_tonH2": squeeze(tank_kg * P["kg_to_tons"]), "turb_mw": squeeze(turb_kw * 1e-3),
        "capital_cost": squeeze(cap_pv + cap_kw + cap_kwh + cap_pem + cap_tank + cap_turb), "capital_cost_pv": squeeze(cap_pv),
        "capital_cost_batt_kw": squeeze(cap_kw), "capital_cost_batt_kwh": squeeze(cap_kwh), "capital_cost_pem": squeeze(cap_pem),
        "capital_cost_tank": squeeze(cap_tank), "capital_cost_turb": squeeze(cap_turb),
        "annual_costs_fixed": squeeze(fixed), "fixed_cost_pv": squeeze(pv_kw * P["pv_op_cost"]), "fixed_cost_pem": squeeze(pem_kw * P["pem_op_cost"]),
        "fixed_cost_tank": squeeze(tank_kg * P["tank_op_cost"]), "fixed_cost_turb": squeeze(turb_kw * P["turbine_op_cost"]),
        "annual_costs_variable": squeeze((pem_var + turb_var).sum(1)), "variable_cost_batt": 0.0,
        "variable_cost_pem": squeeze(pem_var.sum(1)), "variable_cost_turb": squeeze(turb_var.sum(1)),
        "annual_costs_NG": 0.0, "annual_costs_grid": squeeze(grid_cost.sum(1) * 52 / n_weeks),
        "annual_costs_total": squeeze((grid_cost + pem_var + turb_var).sum(1) * 52 / n_weeks),
        "annual_rev_h2": squeeze(h2_rev.sum(1) * 52 / n_weeks), "NPV": squeeze(-r.obj * 1e3), "CO2_lb": 0.0,
        "status": [STATUS_NAMES[int(v)] for v in r.status], "iters": r.iters,
    }
    cf2 = np.broadcast_to(cfs, (N, T))
    df = {
        "Total PV Generation [MW]": (grid + pem + b_in) * 1e-3, "Total Power Output [MW]": (grid + b_out + turb_elec) * 1e-3,
        "PV Power Output [MW]": grid * 1e-3, "PV Power to Battery [MW]": b_in * 1e-3,
        "State of Charge": soc / np.where(batt_kwh > 0, batt_kwh, 1.0)[:, None], "Battery Power Output [MW]": b_out * 1e-3,
        "PV Power to PEM [MW]": pem * 1e-3, "PEM H2 Output [kg]": pem * TP.PEM_ELEC_TO_MOL * P["s_per_ts"] / TP.H2_MOLS_PER_KG,
        "H2 Sales [kg]": to_pipe * P["s_per_ts"] / TP.H2_MOLS_PER_KG, "Turbine H2 Input [kg]": to_turb * P["s_per_ts"] / TP.H2_MOLS_PER_KG,
        "Turbine Power [MW]": turb_elec * 1e-3, "Purchased Power [MW]": purchase * 1e-3, "Sold Power [MW]": sales * 1e-3,
        "Tank Holdup [kg]": holdup / TP.H2_MOLS_PER_KG, "Excess PV [MW]": (pv_kw[:, None] * cf2 - (grid + pem + b_in)) * 1e-3,
        "Battery Reserve [MW]": ser("battery_reserve", True) * 1e-3, "PEM Reserve [MW]": pem * 1e-3,
        "Turbine Reserve [MW]": ser("turbine_reserve", True) * 1e-3, "Load [MW]": np.broadcast_to(load, (N, T)),
        "Grid Income [$]": grid_cost, "H2 Revenue [$]": h2_rev, "Operating Cost [$]": pem_var + turb_var,
    }
    return design_res, df


def record_results(res: PriceTakerResult, k=0):
    """The reference's record_results tuple (wind_battery_LMP.py:272-325) for scenario k."""
    soc = res.series("battery.state_of_charge[0]")[k]
    batt_to_grid = res.series("battery.elec_out[0]")[k] * 1e-3
    wind_to_grid = res.series("splitter.grid_elec[0]")[k] * 1e-3
    wind_to_batt = res.series("battery.elec_in[0]")[k] * 1e-3
    wind_gen = wind_to_grid + wind_to_batt
    lmp = res.lmp[k]
    fixed = res.sizes["wind_kw"][k] * TP.WIND_OP_COST / 8760.0 + res.sizes["batt_kw"][k] * TP.BATT_OP_COST / 8760.0
    elec_revenue = lmp * 1e-3 * (wind_to_grid + batt_to_grid) * 1e3 - fixed
    return (list(soc), list(wind_gen), list(batt_to_grid), list(wind_to_grid), list(wind_to_batt), list(elec_revenue),
            list(lmp), res.sizes["wind_kw"][k] * 1e-3, res.sizes["batt_kw"][k] * 1e-3,
            float(res.annual_revenue[k]), float(res.NPV[k]))
