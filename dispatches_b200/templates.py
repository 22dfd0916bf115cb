"""LP templates of the reference's price-taker flowsheets (reduced / presolved forms).

Each builder mirrors one reference model builder and keeps the reference's Var names for the columns
that survive presolve, so results can be read back by name (record_results, wind_battery_LMP.py:272-325).

Presolve done here once per template (the reference leaves it to CBC on every LP):
  * arcs / ports (w = z, q = i, E = 4P ...) substituted away,
  * fixed Vars become constants, constant lower bounds are shifted to 0,
  * never-binding rows dropped (battery ramp <= 1e8, wind_battery_LMP.py:139-142; nameplate bounds 1e8/1e9),
  * model-level capacity Vars sit at their fixed block values (their cost coefficients are positive),
  * link / periodic equalities substituted (s0[t+1] := s[t]).

Parameter conventions (LPTemplate.instantiate / solver.solve_batch):
  wind_battery(T):        cparams = lmp[T] ($/MWh);  rparams = [wind_kw*cf_0 .. wind_kw*cf_{T-1}, batt_kw, wind_kw]
  wind_battery_pem(T):    cparams = [lmp[T], h2_price];  rparams = [wind_kw*cf_t (T), batt_kw, wind_kw, pem_kw]
  nuclear(T):             cparams = lmp[T];  rparams = [] (design constants baked in)
  fossil_surrogate(T):    cparams = lmp[T];  rparams = []
"""
from __future__ import annotations

import numpy as np

from .lp_template import LPTemplate, TemplateBuilder

# ---- constants of load_parameters.py:24-121 (wind_battery_cost_parameter.json: "moderate", 2023, 4-h)
WIND_CAP_COST = 1308.0
WIND_OP_COST = 41.78
BATT_OP_COST = 31.39
BATT_CAP_COST_KW = 236.365
BATT_CAP_COST_KWH = 254.835
PEM_CAP_COST = 1200.0
PEM_OP_COST = 0.03 * PEM_CAP_COST
PEM_VAR_COST = 0.0
H2_MOLS_PER_KG = 500.0
DURATION = 4.0
ETA_C = ETA_D = 0.95                      # RE_flowsheet.py:151-152
DEGRADATION = 1e-4                        # battery.py:91-95
PEM_ELEC_TO_MOL = 0.00275984              # RE_flowsheet.py:131
PA = ((1 + 0.08) ** 30 - 1) / (0.08 * (1 + 0.08) ** 30)     # load_parameters.py:119-121


def wind_battery(T: int, extant_wind: bool = True) -> LPTemplate:
    """wind_battery_optimize with design_opt=False (wind_battery_LMP.py:172-267; sweep mode of
    run_pricetaker_wind_battery.py:37-58).  Objective = -NPV*1e-5 (:264)."""
    iP, iW = T, T + 1
    B = TemplateBuilder(f"wind_battery_T{T}", Pc=T, Pr=T + 2)
    ann = 52.0 / (T / 168.0)
    k_rev = -1e-5 * PA * ann * 1e-3
    g, i, o, s, e = {}, {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        i[t] = B.var(p + "battery.elec_in[0]", ub=(0.0, {iP: 1.0}))           # battery.py:159-161
        o[t] = B.var(p + "battery.elec_out[0]", ub=(0.0, {iP: 1.0}))          # battery.py:163-165
        # periodic s[T-1] = s0[0] = 0 (:48, :206)  ->  the last state of charge is the constant 0
        s[t] = B.var(p + "battery.state_of_charge[0]", fix=(0.0 if t == T - 1 else None))
        e[t] = B.var(p + "battery.energy_throughput[0]")
        B.cost(g[t], (0.0, {t: k_rev})); B.cost(o[t], (0.0, {t: k_rev}))       # :235-237
    for t in range(T):
        row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}                     # battery.py:145-149
        if t > 0:
            row[s[t - 1]] = -1.0                                              # link :33
        B.eq(f"soc[{t}]", row)
        row = {e[t]: 1.0, i[t]: -0.5, o[t]: -0.5}                              # battery.py:151-153
        if t > 0:
            row[e[t - 1]] = -1.0                                              # link :34
        B.eq(f"throughput[{t}]", row)
        B.le(f"soc_bound[{t}]", {s[t]: 1.0, e[t]: DEGRADATION}, (0.0, {iP: DURATION}))   # battery.py:155-157
        B.le(f"wind[{t}]", {g[t]: 1.0, i[t]: 1.0}, (0.0, {t: 1.0}))           # wind_power.py:120-122 + splitter
    cap = BATT_CAP_COST_KW + BATT_CAP_COST_KWH * DURATION
    B.obj_const((0.0, {iP: 1e-5 * (cap + PA * ann * T * BATT_OP_COST / 8760.0),
                       iW: 1e-5 * ((0.0 if extant_wind else WIND_CAP_COST) + PA * ann * T * WIND_OP_COST / 8760.0)}))
    B.meta.update(kind="wind_battery", T=T, ann=ann)
    t = B.build()
    if True:
        # stage descriptor for the stage kernels (include/dsp_lp.h: dsp_stage_wb_desc): T <= 96 on chip, longer horizons in a workspace
        cn = {n: j for j, n in enumerate(t.col_names)}
        rn = {n: i for i, n in enumerate(t.row_names)}
        col_idx = [[cn.get(f"blk[{k}].fs.splitter.grid_elec[0]", -1), cn.get(f"blk[{k}].fs.battery.elec_in[0]", -1),
                    cn.get(f"blk[{k}].fs.battery.elec_out[0]", -1), cn.get(f"blk[{k}].fs.battery.state_of_charge[0]", -1),
                    cn.get(f"blk[{k}].fs.battery.energy_throughput[0]", -1), cn.get(f"slack:soc_bound[{k}]", -1),
                    cn.get(f"slack:wind[{k}]", -1)] for k in range(T)]
        row_idx = [[rn[f"soc[{k}]"], rn[f"throughput[{k}]"], rn[f"soc_bound[{k}]"], rn[f"wind[{k}]"]] for k in range(T)]
        t.meta["stage_wb"] = dict(T=T, a=ETA_C, binv=1.0 / ETA_D, half=0.5, delta=DEGRADATION, dur=DURATION, k_rev=k_rev,
                                  wcf_off=0, p_off=iP, col_idx=np.array(col_idx, np.int32), row_idx=np.array(row_idx, np.int32))
    return t


def wind_battery_design(T: int, extant_wind: bool = True) -> LPTemplate:
    """wind_battery_optimize with design_opt=True, extant_wind=True (the reference's default_input_params,
    load_parameters.py:123-140; wind_battery_LMP.py:212-216): the battery nameplate power is a decision.

    Formulated the way the reference's MultiPeriodModel does it: one nameplate_power column PER PERIOD with the
    link equalities P[t] = P[t+1] (wind_battery_LMP.py:35), so the constraint matrix stays block banded in time (a
    single global capacity column would be dense; a rank-one (Woodbury) update of the band factor for it was tried and
    is numerically unstable -- DESIGN.md 6b).  battery_system_capacity >= nameplate_power (:219) is tight (positive
    cost), so its capital and O&M cost sit on P[0].  nameplate_energy = 4 P (RE_flowsheet.py:155-156) is substituted.
    rparams = [wind_kw*cf_t (T), unused, wind_kw] (same layout as wind_battery)."""
    if not extant_wind:
        raise NotImplementedError("design_opt with a free wind size puts cf_t into the constraint matrix (not batched)")
    iW = T + 1
    B = TemplateBuilder(f"wind_battery_design_T{T}", Pc=T, Pr=T + 2)
    ann = 52.0 / (T / 168.0)
    k_rev = -1e-5 * PA * ann * 1e-3
    cap = BATT_CAP_COST_KW + BATT_CAP_COST_KWH * DURATION
    g, i, o, s, e, Pn = {}, {}, {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        i[t] = B.var(p + "battery.elec_in[0]")
        o[t] = B.var(p + "battery.elec_out[0]")
        s[t] = B.var(p + "battery.state_of_charge[0]", fix=(0.0 if t == T - 1 else None))
        e[t] = B.var(p + "battery.energy_throughput[0]")
        Pn[t] = B.var(p + "battery.nameplate_power")
        B.cost(g[t], (0.0, {t: k_rev})); B.cost(o[t], (0.0, {t: k_rev}))
    B.cost(Pn[0], 1e-5 * (cap + PA * ann * T * BATT_OP_COST / 8760.0))
    for t in range(T):
        row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}
        if t > 0:
            row[s[t - 1]] = -1.0
        B.eq(f"soc[{t}]", row)
        row = {e[t]: 1.0, i[t]: -0.5, o[t]: -0.5}
        if t > 0:
            row[e[t - 1]] = -1.0
        B.eq(f"throughput[{t}]", row)
        B.le(f"power_bound_in[{t}]", {i[t]: 1.0, Pn[t]: -1.0})
        B.le(f"power_bound_out[{t}]", {o[t]: 1.0, Pn[t]: -1.0})
        B.le(f"soc_bound[{t}]", {s[t]: 1.0, e[t]: DEGRADATION, Pn[t]: -DURATION})
        B.le(f"wind[{t}]", {g[t]: 1.0, i[t]: 1.0}, (0.0, {t: 1.0}))
        if t < T - 1:
            B.eq(f"link_nameplate[{t}]", {Pn[t]: 1.0, Pn[t + 1]: -1.0})
    B.obj_const((0.0, {iW: 1e-5 * (PA * ann * T * WIND_OP_COST / 8760.0)}))
    B.meta.update(kind="wind_battery_design", T=T, ann=ann)
    return B.build()


CF_NOMINAL = 0.35      # nominal capacity factor of the per-problem wind rows (keeps the entry in the pattern; scaling sees it)


def wind_battery_design_free_wind(T: int, cf=None, wind_mw_ub: float = 10000.0) -> LPTemplate:
    """wind_battery_optimize with design_opt=True and extant_wind=False (wind_battery_LMP.py:209-219, :256-263): battery
    AND wind size are decisions.  The wind row  electricity <= system_capacity * cf_t  (wind_power.py:120-122) puts cf_t
    into the constraint matrix, which the batch shares -- so this template is built for ONE capacity-factor series
    (the reference's design runs use the site's series with many price signals) and batched over LMPs only.
    wind_system_capacity >= system_capacity[t] (:218) is tight at the optimum (no other cost on system_capacity[t]); as
    for the battery, one capacity column per period + link equalities keeps the matrix banded.
    cparams = lmp[T];  rparams = [] .

    ``cf=None`` (round 2): the capacity factors become PER-PROBLEM matrix coefficients -- rparams = cf_t - CF_NOMINAL (T values),
    entry -(CF_NOMINAL + rparams[t]) on system_capacity[t] -- so a batch may carry a different wind series per member
    (dsp_lp_template_set_matrix_params; the band kernel re-derives A, A' and the band products per LP)."""
    per_problem = cf is None
    if not per_problem:
        cf = np.asarray(cf, float)
        assert cf.shape == (T,)
    B = TemplateBuilder(f"wind_battery_design_free_wind_T{T}" + ("_cfbatched" if per_problem else ""), Pc=T, Pr=T if per_problem else 0)
    ann = 52.0 / (T / 168.0)
    k_rev = -1e-5 * PA * ann * 1e-3
    cap = BATT_CAP_COST_KW + BATT_CAP_COST_KWH * DURATION
    g, i, o, s, e, Pn, Wn = {}, {}, {}, {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        i[t] = B.var(p + "battery.elec_in[0]")
        o[t] = B.var(p + "battery.elec_out[0]")
        s[t] = B.var(p + "battery.state_of_charge[0]", fix=(0.0 if t == T - 1 else None))
        e[t] = B.var(p + "battery.energy_throughput[0]")
        Pn[t] = B.var(p + "battery.nameplate_power")
        Wn[t] = B.var(p + "windpower.system_capacity", ub=(wind_mw_ub * 1e3 if t == 0 else None))     # :209
        B.cost(g[t], (0.0, {t: k_rev})); B.cost(o[t], (0.0, {t: k_rev}))
    B.cost(Pn[0], 1e-5 * (cap + PA * ann * T * BATT_OP_COST / 8760.0))
    B.cost(Wn[0], 1e-5 * (WIND_CAP_COST + PA * ann * T * WIND_OP_COST / 8760.0))
    for t in range(T):
        row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}
        if t > 0:
            row[s[t - 1]] = -1.0
        B.eq(f"soc[{t}]", row)
        row = {e[t]: 1.0, i[t]: -0.5, o[t]: -0.5}
        if t > 0:
            row[e[t - 1]] = -1.0
        B.eq(f"throughput[{t}]", row)
        B.le(f"power_bound_in[{t}]", {i[t]: 1.0, Pn[t]: -1.0})
        B.le(f"power_bound_out[{t}]", {o[t]: 1.0, Pn[t]: -1.0})
        B.le(f"soc_bound[{t}]", {s[t]: 1.0, e[t]: DEGRADATION, Pn[t]: -DURATION})
        B.le(f"wind[{t}]", {g[t]: 1.0, i[t]: 1.0, Wn[t]: ((-CF_NOMINAL, {t: -1.0}) if per_problem else -float(cf[t]))})
        if t < T - 1:
            B.eq(f"link_nameplate[{t}]", {Pn[t]: 1.0, Pn[t + 1]: -1.0})
            B.eq(f"link_wind[{t}]", {Wn[t]: 1.0, Wn[t + 1]: -1.0})
    B.meta.update(kind="wind_battery_design_free_wind", T=T, ann=ann, per_problem_cf=per_problem)
    return B.build(equilibrate=True)


def wind_battery_rparams(T, cf, wind_mw, batt_mw, pem_mw=None):
    """rparams rows for wind_battery / wind_battery_pem: cf [N,T] or [T]; sizes scalar or [N]."""
    cf = np.atleast_2d(np.asarray(cf, float))
    N = cf.shape[0]
    W = np.broadcast_to(np.asarray(wind_mw, float) * 1e3, (N,))
    P = np.broadcast_to(np.asarray(batt_mw, float) * 1e3, (N,))
    cols = [cf * W[:, None], P[:, None], W[:, None]]
    if pem_mw is not None:
        cols.append(np.broadcast_to(np.asarray(pem_mw, float) * 1e3, (N,))[:, None])
    return np.ascontiguousarray(np.concatenate(cols, axis=1))


def wind_battery_pem(T: int, with_battery: bool = True, extant_wind: bool = True, pem_design: bool = False) -> LPTemplate:
    """wind_battery_pem_optimize with design_opt=False (wind_battery_PEM_LMP.py:180-298).

    Differences from wind_battery: PEM electricity column with H2 revenue (:276), only the initial energy
    throughput is fixed (:217) so the state of charge is periodic (s0[0] = s[T-1], a cyclic link), and
    run_pricetaker_wind_PEM.py:37-41 sweeps with batt_mw = 0 (``with_battery=False`` drops the battery
    columns instead of bounding them by 0).  ``pem_design=True`` is the reference's design_opt="PEM" mode
    (pem_ratio None in run_pricetaker_wind_PEM.py:36-37): pem_system_capacity is a decision -- one capacity column per
    period with link equalities (keeps the matrix banded, see wind_battery_design), its cost on the first copy."""
    iP, iW, iPem = T, T + 1, T + 2
    ih2 = T
    B = TemplateBuilder(f"wind_battery_pem_T{T}" + ("" if with_battery else "_nobatt") + ("_pemdesign" if pem_design else ""),
                        Pc=T + 1, Pr=T + 3)
    ann = 52.0 / (T / 168.0)
    k_rev = -1e-5 * PA * ann * 1e-3
    k_h2 = -1e-5 * PA * ann * PEM_ELEC_TO_MOL / H2_MOLS_PER_KG * 3600.0
    g, i, o, s, e, pe, pc = {}, {}, {}, {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        pe[t] = B.var(p + "pem.electricity[0]", ub=(None if pem_design else (0.0, {iPem: 1.0})))         # :239
        if pem_design:
            pc[t] = B.var(f"pem_system_capacity[{t}]")
        B.cost(g[t], (0.0, {t: k_rev}))
        B.cost(pe[t], (1e-5 * PA * ann * PEM_VAR_COST, {ih2: k_h2}))            # :276, pem var cost :268
        if with_battery:
            i[t] = B.var(p + "battery.elec_in[0]", ub=(0.0, {iP: 1.0}))
            o[t] = B.var(p + "battery.elec_out[0]", ub=(0.0, {iP: 1.0}))
            s[t] = B.var(p + "battery.state_of_charge[0]")
            e[t] = B.var(p + "battery.energy_throughput[0]")
            B.cost(o[t], (0.0, {t: k_rev}))
    for t in range(T):
        wind_row = {g[t]: 1.0, pe[t]: 1.0}
        if with_battery:
            wind_row[i[t]] = 1.0
            row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}
            row[s[(t - 1) % T]] = row.get(s[(t - 1) % T], 0.0) - 1.0            # link + periodic (cyclic)
            B.eq(f"soc[{t}]", row)
            row = {e[t]: 1.0, i[t]: -0.5, o[t]: -0.5}
            if t > 0:
                row[e[t - 1]] = -1.0
            B.eq(f"throughput[{t}]", row)
            B.le(f"soc_bound[{t}]", {s[t]: 1.0, e[t]: DEGRADATION}, (0.0, {iP: DURATION}))
        B.le(f"wind[{t}]", wind_row, (0.0, {t: 1.0}))
        if pem_design:
            B.le(f"pem_max_p[{t}]", {pe[t]: 1.0, pc[t]: -1.0})               # :239
            if t < T - 1:
                B.eq(f"link_pem_capacity[{t}]", {pc[t]: 1.0, pc[t + 1]: -1.0})
    cap = BATT_CAP_COST_KW + BATT_CAP_COST_KWH * DURATION
    if pem_design:
        B.cost(pc[0], 1e-5 * (PEM_CAP_COST + PA * ann * T * PEM_OP_COST / 8760.0))
    om = {iW: 1e-5 * ((0.0 if extant_wind else WIND_CAP_COST) + PA * ann * T * WIND_OP_COST / 8760.0),
          iPem: 0.0 if pem_design else 1e-5 * (PEM_CAP_COST + PA * ann * T * PEM_OP_COST / 8760.0)}
    om[iP] = 1e-5 * (cap + PA * ann * T * BATT_OP_COST / 8760.0)
    B.obj_const((0.0, om))
    B.meta.update(kind="wind_battery_pem", T=T, ann=ann, with_battery=with_battery)
    return B.build()


# ---------------------------------------------------------------------------------------------
MW_H2 = 2.016e-3
NUC_PEM_ELEC_TO_MOL = 0.002527406          # nuclear_flowsheet.py:269


def nuclear(T: int = 48, np_capacity=500.0, pem_capacity=100.0, tank_capacity=5000.0,
            h2_demand=0.35, h2_price=4.0) -> LPTemplate:
    """create_multiperiod_nuclear_model (nuclear_flowsheet_multiperiod_class.py:72-155) as a price-taker LP:
    min sum_t [ operating_cost_t - lmp_t * np_to_grid_t * 1e-3 ]  (operating_cost :149-153)."""
    E = np_capacity * 1e3
    B = TemplateBuilder(f"nuclear_T{T}", Pc=T, Pr=0)
    xp, u, H = {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        xp[t] = B.var(p + "pem.electricity[0]", ub=pem_capacity * 1e3)          # nuclear_flowsheet.py:137-138
        u[t] = B.var(p + "h2_tank.outlet_to_pipeline.flow_mol[0]", ub=h2_demand / MW_H2)   # …_class.py:140-141
        # tank_holdup[t] is tank_holdup_previous[t+1] (link :47-49) whose ub is tank_capacity/mw
        # (nuclear_flowsheet.py:155-156); the last holdup has no successor, hence no upper bound
        H[t] = B.var(p + "h2_tank.tank_holdup[0]", ub=(tank_capacity / MW_H2 if t < T - 1 else None))
        # np_to_grid = E - xp  ->  -lmp*1e-3*(E - xp)
        B.cost(xp[t], (1e-3 * 1.3, {t: 1e-3}))
        B.cost(H[t], MW_H2 * 0.01)
        B.cost(u[t], -MW_H2 * 3600.0 * h2_price)
        B.ocmap[t] += -1e-3 * E
        B.obj_const(E * 1e-3 * 2.3)
    for t in range(T):
        row = {H[t]: 1.0, xp[t]: -3600.0 * NUC_PEM_ELEC_TO_MOL, u[t]: 3600.0}   # hydrogen_tank_simplified.py:177-184
        if t > 0:
            row[H[t - 1]] = -1.0
        B.eq(f"tank_balance[{t}]", row)
    B.meta.update(kind="nuclear", T=T, E=E)
    return B.build(equilibrate=True)          # kW, mol/s and mol columns differ by 1e4: equilibrate (fewer iterations)


def nuclear_report(T: int, pem_capex=400.0, demand=400.0 * 20, vom_pem=0.0, plant_life=30, tax_rate=0.2, discount_rate=0.08,
                   np_mw=400.0) -> LPTemplate:
    """The report's price-taker LP with storage tank and hydrogen turbine (nuclear_case/report/price_taker_analysis.py:116-322):
    build_ne_flowsheet rows (:143-170) reduced to one tank balance per hour --
        np_to_grid = 400 - e,  h2_production = 20 e,  h2_turbine_power = 0.0125 tb,  net_power = 400 - e + 0.0125 tb,
        H[t] - H[t-1] = 20 e[t] - u[t] - tb[t]       (link :175-178, tank_holdup_previous[1] = 0 :377)
    columns e (np_to_electrolyzer <= pem_capacity, :199-203), u (h2_to_pipeline <= demand, :219-220), tb (h2_to_turbine,
    turbine power <= h2_turbine_capacity :209-213), H (tank_holdup <= tank_capacity :204-208).  Objective = -(net_profit -
    capex / cf) of append_* (:239-322; the reference maximises).  The sweep of run_exhaustive_enumeration fixes the three
    capacities (:377-403): they are batch parameters here.
    cparams = [lmp (T), h2_price];  rparams = [pem_capacity MW, tank_capacity kg, h2_turbine_capacity MW]."""
    ih2 = T
    iPem, iTank, iTurb = 0, 1, 2
    k = 1.0 - tax_rate
    cf = (1.0 - (1.0 + discount_rate) ** (-plant_life)) / discount_rate
    B = TemplateBuilder(f"nuclear_report_T{T}", Pc=T + 1, Pr=3)
    e, u, tb, H = {}, {}, {}, {}
    for t in range(T):
        p = f"period[{t + 1}].fs."
        e[t] = B.var(p + "np_to_electrolyzer", ub=(0.0, {iPem: 1.0}))
        u[t] = B.var(p + "h2_to_pipeline", ub=demand)
        tb[t] = B.var(p + "h2_to_turbine", ub=(0.0, {iTurb: 1.0 / 0.0125}))
        H[t] = B.var(p + "tank_holdup", ub=(0.0, {iTank: 1.0}))
        # cash flow (:239-254): h2_price u + lmp net_power - (vom e + 4.25 turbine_power + 2.3 np_power); minimise -(1 - tax) * cash
        B.cost(e[t], (k * vom_pem, {t: k}))                     # -k lmp (400 - e + ...)  ->  + k lmp e
        B.cost(tb[t], (k * 4.25 * 0.0125, {t: -k * 0.0125}))
        B.cost(u[t], (0.0, {ih2: -k}))
        B.ocmap[t] += -k * np_mw
        B.obj_const(k * 2.3 * np_mw)
    for t in range(T):
        row = {H[t]: 1.0, e[t]: -20.0, u[t]: 1.0, tb[t]: 1.0}
        if t > 0:
            row[H[t - 1]] = -1.0
        B.eq(f"tank_mass_balance[{t + 1}]", row)
    # NPV pieces (:274-308): capex = 1000 capex_pem pem + 29*33.3 tank + 1000*947 turbine; fom = 1000 fom_pem pem + 7000 turbine + 120e3*400
    # objective = -(dep + k (cash - fom - dep) - capex / cf),  dep = capex / life
    fom_pem = 0.03 * pem_capex
    capex_coef = {iPem: pem_capex * 1000.0, iTank: 29.0 * 33.3, iTurb: 947.0 * 1000.0}
    fom_coef = {iPem: 1000.0 * fom_pem, iTurb: 1000.0 * 7.0}
    lin = {}
    for i, cc in capex_coef.items():
        lin[i] = lin.get(i, 0.0) - (cc / plant_life) * (1.0 - k) + cc / cf
    for i, fc in fom_coef.items():
        lin[i] = lin.get(i, 0.0) + k * fc
    B.obj_const((k * 120.0 * 1000.0 * np_mw, lin))
    B.meta.update(kind="nuclear_report", T=T, capex_coef=capex_coef, fom_coef=fom_coef, fom_const=120.0 * 1000.0 * np_mw, k=k, cf=cf,
                  plant_life=plant_life, np_mw=np_mw)
    return B.build(equilibrate=True)


# ---------------------------------------------------------------------------------------------
FOSSIL = dict(p_lo=283.0, p_hi=436.0, pprev_lo=284.0, pprev_hi=466.0, hx_lo=10.0, hx_hi=200.0, ramp=60.0,
              salt_total=6739292.0, hot_init=75000.0 + 1103053.48, pprev0=447.66,
              kc=6.5, kd=7.0, eta_c=0.40, eta_d=0.38, fuel=22.0, fixed=6.0)


def fossil_surrogate(T: int = 168, par=None) -> LPTemplate:
    """STRUCTURE-ONLY linear surrogate of the ultra-supercritical plant + molten-salt storage price-taker
    (multiperiod_integrated_storage_usc.py:49-54,75-164,334-342; pricetaker_with_…usc.py:88-107).  The
    reference path is an NLP (IAPWS-95 steam cycle); only its linear inter-period structure is kept --
    parity unpinned, see DESIGN.md."""
    P = dict(FOSSIL); P.update(par or {})
    B = TemplateBuilder(f"fossil_surrogate_T{T}", Pc=T, Pr=0)
    pw, c, d, h = {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        lo = max(P["p_lo"], P["pprev_lo"]) if t < T - 1 else P["p_lo"]         # P[t] is previous_power[t+1]
        pw[t] = B.var(p + "plant_power_out[0]", lb=lo, ub=min(P["p_hi"], P["pprev_hi"]))
        c[t] = B.var(p + "hxc.heat_duty[0]", lb=P["hx_lo"], ub=P["hx_hi"])
        d[t] = B.var(p + "hxd.heat_duty[0]", lb=P["hx_lo"], ub=P["hx_hi"])
        h[t] = B.var(p + "salt_inventory_hot", ub=P["salt_total"], fix=(P["hot_init"] if t == T - 1 else None))
        B.cost(pw[t], (P["fuel"], {t: -1.0}))
        B.cost(c[t], (0.0, {t: P["eta_c"]}))
        B.cost(d[t], (0.0, {t: -P["eta_d"]}))
        B.obj_const(P["fixed"])
    for t in range(T):
        hprev = {h[t - 1]: 1.0} if t > 0 else {}
        hprev_const = 0.0 if t > 0 else P["hot_init"]
        row = {h[t]: 1.0, c[t]: -3600.0 * P["kc"], d[t]: 3600.0 * P["kd"]}
        for j, vv in hprev.items():
            row[j] = -vv
        B.eq(f"hot_balance[{t}]", row, hprev_const)
        row = {d[t]: 3600.0 * P["kd"]}
        for j, vv in hprev.items():
            row[j] = -vv
        B.le(f"discharge_limit[{t}]", row, hprev_const)
        row = {c[t]: 3600.0 * P["kc"]}
        for j, vv in hprev.items():
            row[j] = vv
        B.le(f"charge_limit[{t}]", row, P["salt_total"] - hprev_const)
        if t > 0:
            B.le(f"ramp_up[{t}]", {pw[t]: 1.0, pw[t - 1]: -1.0}, P["ramp"])
            B.le(f"ramp_down[{t}]", {pw[t - 1]: 1.0, pw[t]: -1.0}, P["ramp"])
        else:
            B.le(f"ramp_up[{t}]", {pw[t]: 1.0}, P["ramp"] + P["pprev0"])
            B.le(f"ramp_down[{t}]", {pw[t]: -1.0}, P["ramp"] - P["pprev0"])
    B.meta.update(kind="fossil_surrogate", T=T)
    return B.build(equilibrate=True)          # salt inventories (1e6 kg) next to powers (1e2 MW): must equilibrate


# --------------------------------------------------------------------------------------
# PV + battery + PEM + hydrogen tank + hydrogen turbine, load following with reserves
# --------------------------------------------------------------------------------------
# solar_battery_hydrogen_inputs.py:22-70 (overrides of load_parameters.py; "pem_cap_cost" stays at load_parameters' 1200)
SOLAR = dict(pv_cap_cost=WIND_CAP_COST, pv_op_cost=WIND_OP_COST, batt_cap_cost_kw=236.36 * 0.5, batt_cap_cost_kwh=254.83 * 0.5,
             pem_cap_cost=PEM_CAP_COST, pem_op_cost=47.9, pem_var_cost=1.3e-3, tank_cap_cost_per_kg=500.0, tank_op_cost=85.0,
             turbine_cap_cost=1320.0, turbine_op_cost=11.65, turbine_var_cost=3e-3, h2_price_per_kg=2.5,
             capacity_requirement=100.0, capacity_credit_battery=0.33, turbine_min_mw=0.0, turbine_ramp_mw_per_min=100.0,
             h2_turb_conv=0.39 * 33.391, flow_mol_ub=1e5, kg_to_tons=0.00110231, s_per_ts=3600.0)


def solar_battery_hydrogen(T: int, batt_mw=0.0, batt_mwh=0.0, pem_mw=0.0, tank_kg=None, turb_mw=100.0, reserve_mw=100.0,
                           max_sales=1000.0, max_purchases=1000.0, par=None) -> LPTemplate:
    """pv_battery_hydrogen_optimize with design_opt=False (solar_battery_hydrogen.py:375-457; h2_blend_ratio = 1): PV + battery
    + PEM + hydrogen tank + hydrogen turbine following a load with a reserve requirement, grid purchases / sales at the LMP.
    Objective = -NPV*1e-3 (:372).  Sizes are template constants (the reference fixes them, :222-228); the batch runs over
    cparams = lmp[T] and rparams = [pv_kw*cf_t (T), load_kw_t (T), pv_kw].

    Presolve: arcs substituted (w = z, p = pe, q = i, tank inlet = PEM outlet); nameplate power / energy at their fixed values;
    energy_throughput dropped (degradation_rate = 0, :173, leaves it in no other row); link equalities substituted, the periodic
    pairs (:58-61) make state of charge and tank holdup CYCLIC in time; grid_sales - grid_purchase <= max_sales is implied by the
    bounds (:355-360); the turbine ramp rows (:323-324) are dropped when the ramp limit exceeds the turbine capacity; the
    capacity requirement (:352) involves constants only and is checked here."""
    P = dict(SOLAR); P.update(par or {})
    if tank_kg is None:
        tank_kg = P["capacity_requirement"] * 1e3 / P["h2_turb_conv"]           # inputs.py:86
    Bc, Be, Pc, Tc = batt_mw * 1e3, batt_mwh * 1e3, pem_mw * 1e3, turb_mw * 1e3
    if Bc * P["capacity_credit_battery"] + Tc < P["capacity_requirement"] * 1e3 - 1e-9:
        raise ValueError("capacity requirement (solar_battery_hydrogen.py:352) cannot be met by the fixed sizes")
    if not (0.5 * Bc - 1e-9 <= Be <= 8.0 * Bc + 1e-9):
        raise ValueError("battery duration outside 0.5 .. 8 hours (solar_battery_hydrogen.py:234-235)")
    reserve = np.broadcast_to(np.asarray(reserve_mw, float), (T,))
    k_turb = P["s_per_ts"] / H2_MOLS_PER_KG * P["h2_turb_conv"]                  # kW per mol/s sent to the turbine
    k_res = P["h2_turb_conv"] / H2_MOLS_PER_KG                                  # kW of reserve per mol of holdup
    ramp = P["turbine_ramp_mw_per_min"] * 1e3
    iA, iL, iPV = 0, T, 2 * T
    B = TemplateBuilder(f"solar_battery_hydrogen_T{T}", Pc=T, Pr=2 * T + 1)
    ann = 52.143 / (T / 168.0)
    kk = 1e-3 * PA * ann
    w, g, pe, i, o, s, tt, tp, hd, gp, gs, tr, br = ({} for _ in range(13))
    have_batt, have_pem = Bc > 0.0, Pc > 0.0
    for t in range(T):
        p = f"blk[{t}].fs."
        w[t] = B.var(p + "pv.electricity[0]", ub=(0.0, {iA + t: 1.0}))                       # solar_pv.py:82-84
        g[t] = B.var(p + "splitter.grid_elec[0]")
        if have_pem:
            pe[t] = B.var(p + "pem.electricity[0]", ub=min(Pc, P["flow_mol_ub"] / PEM_ELEC_TO_MOL))     # pem_max_p :229
            B.cost(pe[t], kk * P["pem_var_cost"])
        if have_batt:
            i[t] = B.var(p + "battery.elec_in[0]", ub=Bc)
            o[t] = B.var(p + "battery.elec_out[0]", ub=Bc)
            s[t] = B.var(p + "battery.state_of_charge[0]", ub=Be)
            br[t] = B.var(f"blk[{t}].battery_reserve", ub=Bc)                                # battery_reserve_lb1
        tt[t] = B.var(p + "h2_tank.outlet_to_turbine.flow_mol[0]", lb=P["turbine_min_mw"] * 1e3 / k_turb,
                      ub=min(P["flow_mol_ub"], Tc / k_turb))                                # h2_turbine_pmin :159, turb_max_p :231
        tp[t] = B.var(p + "h2_tank.outlet_to_pipeline.flow_mol[0]", ub=P["flow_mol_ub"])
        hd[t] = B.var(p + "h2_tank.tank_holdup[0]", ub=tank_kg * H2_MOLS_PER_KG)             # tank_max_p :230
        gp[t] = B.var(f"blk[{t}].grid_purchase", ub=max_purchases * 1e3)
        gs[t] = B.var(f"blk[{t}].grid_sales", ub=max_sales * 1e3)
        tr[t] = B.var(f"blk[{t}].turbine_reserve")
        B.cost(gs[t], (0.0, {t: -kk * 1e-3})); B.cost(gp[t], (0.0, {t: kk * 1e-3}))           # grid_cost :361
        B.cost(tt[t], kk * P["turbine_var_cost"] * k_turb)
        B.cost(tp[t], -kk * P["h2_price_per_kg"] / H2_MOLS_PER_KG * P["s_per_ts"])           # hydrogen_revenue :354
    for t in range(T):
        tm = (t - 1) % T
        row = {w[t]: 1.0, g[t]: -1.0}                                                       # elec_splitter.py:115-117
        if have_pem:
            row[pe[t]] = -1.0
        if have_batt:
            row[i[t]] = -1.0
        B.eq(f"split[{t}]", row)
        if have_batt:
            row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}                               # battery.py:145-149, links :44 / :59
            row[s[tm]] = row.get(s[tm], 0.0) - 1.0
            B.eq(f"soc[{t}]", row)
            B.le(f"battery_reserve_lb2[{t}]", {br[t]: 1.0, s[t]: -1.0})
        row = {hd[t]: 1.0, tp[t]: P["s_per_ts"], tt[t]: P["s_per_ts"]}                        # hydrogen_tank_simplified.py:177-184
        row[hd[tm]] = row.get(hd[tm], 0.0) - 1.0
        if have_pem:
            row[pe[t]] = -P["s_per_ts"] * PEM_ELEC_TO_MOL
        B.eq(f"tank[{t}]", row)
        row = {g[t]: 1.0, tt[t]: k_turb, gp[t]: 1.0, gs[t]: -1.0}                             # meet_load :331
        if have_batt:
            row[o[t]] = 1.0
        B.eq(f"meet_load[{t}]", row, (0.0, {iL + t: 1.0}))
        B.le(f"turbine_reserve_lb1[{t}]", {tr[t]: 1.0, hd[t]: -k_res})
        B.le(f"turbine_reserve_lb2[{t}]", {tr[t]: 1.0, tt[t]: k_turb}, Tc)
        r1 = (max(reserve[max(t - 1, 0):t]) if t > 0 else reserve[0]) * 1e3                   # :347-348
        row = {tr[t]: -1.0, w[t]: 1.0}                                                      # min_reserve :349
        if have_batt:
            row[br[t]] = -1.0
        if have_pem:
            row[pe[t]] = -1.0
        B.le(f"min_reserve[{t}]", row, (-r1, {iA + t: 1.0}))
        if ramp < Tc and T > 1:
            B.le(f"energy_down_ramp[{t}]", {tt[tm]: k_turb, tt[t]: -k_turb}, ramp)
            B.le(f"energy_up_ramp[{t}]", {tt[t]: k_turb, tt[tm]: -k_turb}, ramp)
    cap = (P["batt_cap_cost_kw"] * Bc + P["batt_cap_cost_kwh"] * Be + P["pem_cap_cost"] * Pc + P["tank_cap_cost_per_kg"] * tank_kg)
    fixed = Pc * P["pem_op_cost"] + tank_kg * P["tank_op_cost"] + Tc * P["turbine_op_cost"]
    B.obj_const((1e-3 * (cap + PA * fixed), {iPV: 1e-3 * PA * P["pv_op_cost"]}))
    # The reference sizes the tank EXACTLY for the reserve it must back (inputs.py:86): at night turbine_reserve >= reserve forces the
    # holdup to its upper bound, the feasible set has no strict interior in those columns and the interior-point iterates crawl
    # (with the default proximal term 1e-8 an occasional LP needs over 100 iterations, with 1e-7 none needs more than about 15:
    # tools/gpu_solar_diag.py compares the two) -- the solver reads this value unless the caller passes its own.
    B.meta.update(kind="solar_battery_hydrogen", T=T, ann=ann, capital_cost=cap, k_turb=k_turb, tank_kg=tank_kg,
                  sizes=dict(batt_kw=Bc, batt_kwh=Be, pem_kw=Pc, turb_kw=Tc), reg_primal=1e-7)
    return B.build(equilibrate=True)         # holdups (1e6 mol) next to powers (1e5 kW) and flows (1e2 mol/s)


SOLAR_SIZE_COLUMNS = ("pv_add_system_capacity", "battery_system_capacity", "battery_system_energy", "pem_system_capacity",
                      "h2_tank_size", "turb_system_capacity")


def solar_battery_hydrogen_design(T: int, pv_cfs, pv_mw=0.0, turb_mw=0.0, reserve_mw=100.0, max_sales=1000.0, max_purchases=1000.0,
                                  par=None) -> LPTemplate:
    """pv_battery_hydrogen_optimize with design_opt=True (size_constraints, solar_battery_hydrogen.py:205-236): the six sizes
    (added PV, battery power / energy, PEM, tank, turbine) are columns of their own, each in a ``<=`` row of every period.  Those six
    columns make A A' dense (half bandwidth 225 at T = 24), so the band kernels cannot take this template;
    ``lp_template.find_linking_columns`` finds exactly these six, and without them the half bandwidth is 31 (DESIGN §2 row (f)).
    The PV capacity factors multiply the added-PV column, so the PV series is part of the template; the batch runs over
    cparams = lmp[T] and rparams = load_kw[T].

    Presolve against the raw LP: arcs substituted as in ``solar_battery_hydrogen``; the per-period nameplate power / energy and PV
    capacity copies replaced by the size columns they are bounded by (nothing else prices them, so they sit at the size); the
    capacity requirement (:352, repeated in every period) kept once; pv.electricity substituted by the splitter balance; the two
    turbine ramp rows of a period as one ranged row; turb_max_p (:231) dropped, turbine_reserve_lb2 implies it (reserve >= 0); the
    size bounds of 1e7 / 1e8 kW and the hydrogen-flow bound of the PEM (3.6e7 kW) dropped: they never bind at a size anyone pays for,
    and next to kW-scale flows they would set the scale of the whole LP; the cyclic chain of nameplate-power links (:47, :61) is gone with
    the copies, so none of its redundant links remains; grid_sales - grid_purchase <= max_sales is implied by the bounds."""
    P = dict(SOLAR); P.update(par or {})
    cf = np.asarray(pv_cfs, float).reshape(T)
    reserve = np.broadcast_to(np.asarray(reserve_mw, float), (T,))
    pv_base, turb_base = pv_mw * 1e3, turb_mw * 1e3
    k_turb = P["s_per_ts"] / H2_MOLS_PER_KG * P["h2_turb_conv"]
    k_res = P["h2_turb_conv"] / H2_MOLS_PER_KG
    k_pem = P["s_per_ts"] * PEM_ELEC_TO_MOL
    ramp = P["turbine_ramp_mw_per_min"] * 1e3
    fmax = P["flow_mol_ub"]
    B = TemplateBuilder(f"solar_battery_hydrogen_design_T{T}", Pc=T, Pr=T)
    ann = 52.143 / (T / 168.0)
    kk = 1e-3 * PA * ann
    Va = B.var("pv_add_system_capacity")
    Bc = B.var("battery_system_capacity")
    Be = B.var("battery_system_energy")
    Pc = B.var("pem_system_capacity")
    Ts = B.var("h2_tank_size")
    Tc = B.var("turb_system_capacity", lb=turb_base)
    B.cost(Va, 1e-3 * (P["pv_cap_cost"] + PA * P["pv_op_cost"]))
    B.cost(Bc, 1e-3 * P["batt_cap_cost_kw"]); B.cost(Be, 1e-3 * P["batt_cap_cost_kwh"])
    B.cost(Pc, 1e-3 * (P["pem_cap_cost"] + PA * P["pem_op_cost"]))
    B.cost(Ts, 1e-3 * (P["tank_cap_cost_per_kg"] + PA * P["tank_op_cost"]))
    B.cost(Tc, 1e-3 * (P["turbine_cap_cost"] + PA * P["turbine_op_cost"]))
    B.obj_const(1e-3 * (PA * pv_base * P["pv_op_cost"] - P["turbine_cap_cost"] * turb_base))
    g, pe, i, o, s, br, tt, tp, hd, gp, gs, tr = ({} for _ in range(12))
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        pe[t] = B.var(p + "pem.electricity[0]")
        i[t] = B.var(p + "battery.elec_in[0]")
        o[t] = B.var(p + "battery.elec_out[0]")
        s[t] = B.var(p + "battery.state_of_charge[0]")
        br[t] = B.var(f"blk[{t}].battery_reserve")
        tt[t] = B.var(p + "h2_tank.outlet_to_turbine.flow_mol[0]", lb=P["turbine_min_mw"] * 1e3 / k_turb, ub=fmax)
        tp[t] = B.var(p + "h2_tank.outlet_to_pipeline.flow_mol[0]", ub=fmax)
        hd[t] = B.var(p + "h2_tank.tank_holdup[0]")
        gp[t] = B.var(f"blk[{t}].grid_purchase", ub=max_purchases * 1e3)
        gs[t] = B.var(f"blk[{t}].grid_sales", ub=max_sales * 1e3)
        tr[t] = B.var(f"blk[{t}].turbine_reserve")
        B.cost(gs[t], (0.0, {t: -kk * 1e-3})); B.cost(gp[t], (0.0, {t: kk * 1e-3}))
        B.cost(pe[t], kk * P["pem_var_cost"])
        B.cost(tt[t], kk * P["turbine_var_cost"] * k_turb)
        B.cost(tp[t], -kk * P["h2_price_per_kg"] / H2_MOLS_PER_KG * P["s_per_ts"])
    for t in range(T):
        tm = (t - 1) % T
        pv = {g[t]: 1.0, pe[t]: 1.0, i[t]: 1.0}                       # pv.electricity = grid + PEM + battery (elec_splitter.py:115-117)
        B.le(f"pv_max[{t}]", {**pv, Va: -cf[t]} if cf[t] != 0.0 else pv, cf[t] * pv_base)                      # solar_pv.py:82-84
        row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}
        row[s[tm]] = row.get(s[tm], 0.0) - 1.0
        B.eq(f"soc[{t}]", row)
        B.le(f"soc_max[{t}]", {s[t]: 1.0, Be: -1.0})                                         # battery.py:155-157, :225-226
        B.le(f"charge_max[{t}]", {i[t]: 1.0, Bc: -1.0})
        B.le(f"discharge_max[{t}]", {o[t]: 1.0, Bc: -1.0})
        B.le(f"battery_reserve_lb1[{t}]", {br[t]: 1.0, Bc: -1.0})
        B.le(f"battery_reserve_lb2[{t}]", {br[t]: 1.0, s[t]: -1.0})
        B.le(f"pem_max_p[{t}]", {pe[t]: 1.0, Pc: -1.0})                                      # :229
        row = {hd[t]: 1.0, tp[t]: P["s_per_ts"], tt[t]: P["s_per_ts"], pe[t]: -k_pem}
        row[hd[tm]] = row.get(hd[tm], 0.0) - 1.0
        B.eq(f"tank[{t}]", row)
        B.le(f"tank_max_p[{t}]", {hd[t]: 1.0 / H2_MOLS_PER_KG, Ts: -1.0})                    # :230
        B.eq(f"meet_load[{t}]", {g[t]: 1.0, o[t]: 1.0, tt[t]: k_turb, gp[t]: 1.0, gs[t]: -1.0}, (0.0, {t: 1.0}))
        B.le(f"turbine_reserve_lb1[{t}]", {tr[t]: 1.0, hd[t]: -k_res})
        B.le(f"turbine_reserve_lb2[{t}]", {tr[t]: 1.0, tt[t]: k_turb, Tc: -1.0})
        r1 = (max(reserve[max(t - 1, 0):t]) if t > 0 else reserve[0]) * 1e3
        row = {br[t]: -1.0, tr[t]: -1.0, g[t]: 1.0, i[t]: 1.0}                       # PV headroom C cf - w with w substituted
        if cf[t] != 0.0:
            row[Va] = -cf[t]
        B.le(f"min_reserve[{t}]", row, -r1 + cf[t] * pv_base)
        if T > 1:                                                                            # both ramp rows (:323-324) as one ranged row
            rr = B.var(f"ramp_range[{t}]", ub=2.0 * ramp)
            B.eq(f"energy_ramp[{t}]", {tt[t]: k_turb, tt[tm]: -k_turb, rr: 1.0}, ramp)
    B.le("battery_min_duration", {Bc: 0.5, Be: -1.0})                                        # :234-235
    B.le("battery_max_duration", {Be: 1.0, Bc: -8.0})
    B.le("capacity_requirement", {Bc: -P["capacity_credit_battery"], Tc: -1.0}, -P["capacity_requirement"] * 1e3)
    B.meta.update(kind="solar_battery_hydrogen_design", T=T, ann=ann, k_turb=k_turb, pv_base=pv_base, turb_base=turb_base, pv_cfs=cf.copy())
    # not equilibrated: the six size columns sit in rows of every period, and the geometric-mean row / column scaling then stretches
    # the bounds and costs over 1e-8 .. 1e11 (the interior-point iterates diverge); in kW, mol and $ the LP solves in about 22 iterations
    return B.build(equilibrate=False)


def solar_rparams(T, pv_cfs, pv_mw, load_mw):
    """rparams rows of solar_battery_hydrogen: [pv_kw*cf_t (T), load_kw_t (T), pv_kw]; pv_cfs / load_mw [T] or [N, T], pv_mw scalar or [N]"""
    cf = np.atleast_2d(np.asarray(pv_cfs, float)); ld = np.atleast_2d(np.asarray(load_mw, float))
    pv = np.atleast_1d(np.asarray(pv_mw, float)) * 1e3
    N = max(cf.shape[0], ld.shape[0], pv.size)
    out = np.empty((N, 2 * T + 1))
    out[:, :T] = pv[:, None] * cf
    out[:, T:2 * T] = ld * 1e3
    out[:, 2 * T] = pv
    return out


# --------------------------------------------------------------------------------------
# double-loop operation model: tracking / bidding LPs (SURVEY.md §8(f)-2)
# --------------------------------------------------------------------------------------
BATT_REP_COST_KWH = BATT_CAP_COST_KW * 0.5 / 4.0     # load_parameters.py:48
LARGE_PENALTY = 1e4                                  # idaes-pse 2.0 Tracker deviation / Bidder underbid penalty


def wind_battery_operation(T: int, mode: str, n_tracking_hour: int = 1) -> LPTemplate:
    """Operation model of wind_battery_double_loop.py:27-83,160-171 (sizes fixed, initial SoC / throughput fixed, no
    periodic row) with the objective and extra rows of the IDAES double-loop object that owns it:

      mode "tracker"    Tracker.track_market_dispatch: min tot_cost + pen_t (under_t + over_t),
                        P_T[t] + under_t == dispatch_t + over_t
      mode "bidder_da"  SelfScheduler / Bidder day-ahead problem (one scenario): max da*Pda + rt*(P_T - Pda) - tot_cost,
                        Pda_t <= P_T[t]
      mode "bidder_rt"  the real-time problem: Pda fixed to the cleared day-ahead dispatch, underbid_t >= 0 at 1e4 $/MW
                        (the constant (da-rt)*Pda is added back by the host, dispatches_b200/double_loop.py)

    Internal columns are in kW (the reference's unit for the block Vars); the MW quantities of the IDAES layer
    (under/over, day_ahead_power, underbid) are carried in kW too and scaled on read-back.
    rparams = [wind_kw*cf_t (T), batt_kw, energy_kwh, soc0_kwh, thr0_kwh, wind_kw, dispatch_or_da_dispatch_MW_t (T)]
    cparams = tracker: [wind_waste_penalty];  bidder_*: [da_t (T), rt_t (T), wind_waste_penalty]   ($/MWh, $/MW)
    """
    assert mode in ("tracker", "bidder_da", "bidder_rt")
    iP, iE, iS0, iE0, iW, iD = T, T + 1, T + 2, T + 3, T + 4, T + 5
    Pc = 1 if mode == "tracker" else 2 * T + 1
    iPen = Pc - 1
    B = TemplateBuilder(f"wind_battery_{mode}_T{T}", Pc=Pc, Pr=2 * T + 5)
    kdeg = DEGRADATION * BATT_REP_COST_KWH
    g, i, o, s, e, waste = {}, {}, {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        i[t] = B.var(p + "battery.elec_in[0]", ub=(0.0, {iP: 1.0}))           # battery.py:159-161
        o[t] = B.var(p + "battery.elec_out[0]", ub=(0.0, {iP: 1.0}))          # battery.py:163-165
        s[t] = B.var(p + "battery.state_of_charge[0]")
        e[t] = B.var(p + "battery.energy_throughput[0]")
        waste[t] = B.var(f"wind_waste_kw[{t}]")                               # double_loop.py:169
        B.cost(waste[t], (0.0, {iPen: 1e-3}))                                 # :165,171
    B.cost(e[T - 1], kdeg)                                                    # sum_t var_cost telescopes (wind_battery_LMP.py:67-70)
    B.obj_const((0.0, {iE0: -kdeg, iW: T * WIND_OP_COST / 8760.0}))           # :61-64
    for t in range(T):
        row = {s[t]: 1.0, i[t]: -ETA_C, o[t]: 1.0 / ETA_D}                     # battery.py:145-149
        if t > 0:
            row[s[t - 1]] = -1.0
        B.eq(f"soc[{t}]", row, (0.0, {iS0: 1.0}) if t == 0 else 0.0)          # double_loop.py:76-77,190-191
        row = {e[t]: 1.0, i[t]: -0.5, o[t]: -0.5}                              # battery.py:151-153
        if t > 0:
            row[e[t - 1]] = -1.0
        B.eq(f"throughput[{t}]", row, (0.0, {iE0: 1.0}) if t == 0 else 0.0)   # double_loop.py:193-196
        B.le(f"soc_bound[{t}]", {s[t]: 1.0, e[t]: DEGRADATION}, (0.0, {iE: 1.0}))    # battery.py:155-157
        B.eq(f"wind[{t}]", {g[t]: 1.0, i[t]: 1.0, waste[t]: 1.0}, (0.0, {t: 1.0}))   # wind_power.py:120-122 + splitter
        if mode == "tracker":
            un = B.var(f"power_underdelivered_kw[{t}]"); ov = B.var(f"power_overdelivered_kw[{t}]")
            pen = LARGE_PENALTY if t < n_tracking_hour else LARGE_PENALTY / max(1, T - n_tracking_hour)
            B.cost(un, pen * 1e-3); B.cost(ov, pen * 1e-3)
            B.eq(f"tracking_dispatch[{t}]", {g[t]: 1.0, o[t]: 1.0, un: 1.0, ov: -1.0}, (0.0, {iD + t: 1e3}))
        else:
            B.cost(g[t], (0.0, {T + t: -1e-3})); B.cost(o[t], (0.0, {T + t: -1e-3}))
            if mode == "bidder_da":
                da = B.var(f"day_ahead_power_kw[{t}]")
                B.cost(da, (0.0, {t: -1e-3, T + t: 1e-3}))
                B.le(f"day_ahead_power_ub[{t}]", {da: 1.0, g[t]: -1.0, o[t]: -1.0})
            else:
                ub = B.var(f"real_time_underbid_power_kw[{t}]"); sp_ = B.var(f"surplus_kw[{t}]")
                B.cost(ub, LARGE_PENALTY * 1e-3)
                B.eq(f"day_ahead_power_ub[{t}]", {g[t]: 1.0, o[t]: 1.0, ub: 1.0, sp_: -1.0}, (0.0, {iD + t: 1e3}))
    B.meta.update(kind="wind_battery_operation", mode=mode, T=T, n_tracking_hour=n_tracking_hour)
    return B.build()


def wind_battery_operation_rparams(T, cf, wind_mw, batt_mw, energy_mwh, soc0_kwh=0.0, thr0_kwh=0.0, signal_mw=None):
    """rparams rows of wind_battery_operation: cf [N,T] or [T]; the rest scalar or [N]; signal_mw [N,T] / [T] / None."""
    cf = np.atleast_2d(np.asarray(cf, float))
    N = cf.shape[0]
    col = lambda v, k=1.0: np.broadcast_to(np.asarray(v, float) * k, (N,))[:, None]
    W = col(wind_mw, 1e3)
    sig = np.zeros((N, T)) if signal_mw is None else np.broadcast_to(np.atleast_2d(np.asarray(signal_mw, float)), (N, T))
    return np.ascontiguousarray(np.concatenate(
        [cf * W, col(batt_mw, 1e3), col(energy_mwh, 1e3), col(soc0_kwh), col(thr0_kwh), W, sig], axis=1))


NUC_NP_CAPACITY_MW = 500.0       # flowsheet_options of create_multiperiod_nuclear_model (…_class.py:97-102)


def nuclear_operation(T: int, mode: str, n_tracking_hour: int = 1, np_capacity=NUC_NP_CAPACITY_MW, pem_capacity=100.0,
                      tank_capacity=5000.0, h2_demand=0.35) -> LPTemplate:
    """MultiPeriodNuclear's operation model (nuclear_flowsheet_multiperiod_class.py:72-155, :190-215) under the Tracker /
    Bidder objectives (see wind_battery_operation).  P_T = np_to_grid * 1e-3 = (E - pem.electricity) * 1e-3.
    rparams = [tank_holdup_previous of block 0 (mol), dispatch_or_da_dispatch_MW_t (T)]
    cparams = tracker: [h2_price];  bidder_*: [da_t (T), rt_t (T), h2_price]"""
    assert mode in ("tracker", "bidder_da", "bidder_rt")
    E = np_capacity * 1e3
    Pc = 1 if mode == "tracker" else 2 * T + 1
    iH2, iH0, iD = Pc - 1, 0, 1
    B = TemplateBuilder(f"nuclear_{mode}_T{T}", Pc=Pc, Pr=T + 1)
    xp, u, H = {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        xp[t] = B.var(p + "pem.electricity[0]", ub=pem_capacity * 1e3)
        u[t] = B.var(p + "h2_tank.outlet_to_pipeline.flow_mol[0]", ub=h2_demand / MW_H2)
        H[t] = B.var(p + "h2_tank.tank_holdup[0]", ub=(tank_capacity / MW_H2 if t < T - 1 else None))
        B.cost(xp[t], 1e-3 * 1.3); B.cost(H[t], MW_H2 * 0.01)                # operating_cost :149-153
        B.cost(u[t], (0.0, {iH2: -MW_H2 * 3600.0}))
        B.obj_const(E * 1e-3 * 2.3)
    for t in range(T):
        row = {H[t]: 1.0, xp[t]: -3600.0 * NUC_PEM_ELEC_TO_MOL, u[t]: 3600.0}
        if t > 0:
            row[H[t - 1]] = -1.0
        B.eq(f"tank_balance[{t}]", row, (0.0, {iH0: 1.0}) if t == 0 else 0.0)  # :203, :233-235
        if mode == "tracker":
            un = B.var(f"power_underdelivered_kw[{t}]"); ov = B.var(f"power_overdelivered_kw[{t}]")
            pen = LARGE_PENALTY if t < n_tracking_hour else LARGE_PENALTY / max(1, T - n_tracking_hour)
            B.cost(un, pen * 1e-3); B.cost(ov, pen * 1e-3)
            B.eq(f"tracking_dispatch[{t}]", {xp[t]: -1.0, un: 1.0, ov: -1.0}, (-E, {iD + t: 1e3}))
        else:
            B.cost(xp[t], (0.0, {T + t: 1e-3})); B.ocmap[T + t] += -1e-3 * E   # -rt * (E - xp) * 1e-3
            if mode == "bidder_da":
                da = B.var(f"day_ahead_power_kw[{t}]")
                B.cost(da, (0.0, {t: -1e-3, T + t: 1e-3}))
                B.le(f"day_ahead_power_ub[{t}]", {da: 1.0, xp[t]: 1.0}, E)
            else:
                ub = B.var(f"real_time_underbid_power_kw[{t}]"); sp_ = B.var(f"surplus_kw[{t}]")
                B.cost(ub, LARGE_PENALTY * 1e-3)
                B.eq(f"day_ahead_power_ub[{t}]", {xp[t]: -1.0, ub: 1.0, sp_: -1.0}, (-E, {iD + t: 1e3}))
    B.meta.update(kind="nuclear_operation", mode=mode, T=T, E=E, n_tracking_hour=n_tracking_hour)
    return B.build(equilibrate=True)


def wind_pem_operation(T: int, mode: str = "tracker", n_tracking_hour: int = 1) -> LPTemplate:
    """MultiPeriodWindPEM's operation model (wind_PEM_double_loop.py:25-172; battery size 0) under the Tracker objective.
    pem_system_capacity is a free non-negative Var of that model (:69-73): one copy per period + link equalities (banded).
    Its bidder is parametrised (no LP), so "tracker" is the only mode.
    rparams = [wind_kw*cf_t (T), wind_kw, dispatch_MW_t (T)];  cparams = [wind_waste weight ($/kW, 1 in the reference)]"""
    assert mode == "tracker"
    iW, iD = T, T + 1
    B = TemplateBuilder(f"wind_pem_tracker_T{T}", Pc=1, Pr=2 * T + 1)
    g, pe, waste, cap = {}, {}, {}, {}
    for t in range(T):
        p = f"blk[{t}].fs."
        g[t] = B.var(p + "splitter.grid_elec[0]")
        pe[t] = B.var(p + "pem.electricity[0]")
        waste[t] = B.var(f"wind_waste_kw[{t}]")
        cap[t] = B.var(f"pem_system_capacity[{t}]")
        B.cost(waste[t], (0.0, {0: 1.0}))                                    # :172
        B.cost(pe[t], PEM_VAR_COST)
        B.cost(cap[t], PEM_OP_COST / 8760.0)                                 # :171, once per period
    B.obj_const((0.0, {iW: T * WIND_OP_COST / 8760.0}))                       # :170
    for t in range(T):
        B.eq(f"wind[{t}]", {g[t]: 1.0, pe[t]: 1.0, waste[t]: 1.0}, (0.0, {t: 1.0}))
        B.le(f"pem_max_p[{t}]", {pe[t]: 1.0, cap[t]: -1.0})                  # :73
        un = B.var(f"power_underdelivered_kw[{t}]"); ov = B.var(f"power_overdelivered_kw[{t}]")
        pen = LARGE_PENALTY if t < n_tracking_hour else LARGE_PENALTY / max(1, T - n_tracking_hour)
        B.cost(un, pen * 1e-3); B.cost(ov, pen * 1e-3)
        B.eq(f"tracking_dispatch[{t}]", {g[t]: 1.0, un: 1.0, ov: -1.0}, (0.0, {iD + t: 1e3}))
        if t < T - 1:
            B.eq(f"link_pem_capacity[{t}]", {cap[t]: 1.0, cap[t + 1]: -1.0})
    B.meta.update(kind="wind_pem_operation", mode=mode, T=T, n_tracking_hour=n_tracking_hour)
    return B.build()
