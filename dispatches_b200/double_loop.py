"""Double-loop (bidding / tracking) LPs on the batched CUDA solver -- SURVEY.md §8(f)-2.

Host-side mirror of the reference's ``MultiPeriodWindBattery`` (case_studies/renewables_case/
wind_battery_double_loop.py:104-352) and of the three IDAES objects that own its LPs in the reference's tests
(case_studies/renewables_case/tests/test_multiperiod_wind_battery_doubleloop.py:47-111, :114-175, :178-252):
``Tracker``, ``SelfScheduler`` / ``Bidder`` and the ``Backcaster`` price forecaster.  idaes-pse is not vendored in the
reference; the formulation of those objects is restated (see oracle/double_loop.py for the anchoring on the
reference's known answers) and only the part of their interface the reference exercises is provided.

Same names and argument meaning as the reference; the one extension is batching: ``wind_capacity_factors`` may be
[N, L] and the sizes [N] (N independent simulations advanced in lock step -- the reference runs one per process), and
``market_dispatch`` / price histories may carry a leading batch axis.  Every LP goes through
``BatchLPSolver.solve_host`` (C-ABI ``dsp_lp_solve_batch_host``); there is no CPU fallback.
"""
from __future__ import annotations

import dataclasses
from collections import deque

import numpy as np

from . import templates as TP
from .solver import BatchLPSolver, OPTIMAL

_SOLVERS = {}


_FAMILIES = {"wind_battery": TP.wind_battery_operation, "nuclear": TP.nuclear_operation, "wind_pem": TP.wind_pem_operation}


def _lp_solve(mode, T, cparams, rparams, n_tracking_hour=1, options=None, family="wind_battery"):
    """One batched solve of the operation template; returns (obj [N], status [N], columns {name: [N,T]}).  options["crossover"]:
    the columns come from a vertex of each LP (BatchLPSolver.crossover), as a simplex solver such as the reference's CBC returns
    them; an LP whose crossover does not end OPTIMAL keeps its interior-point solution."""
    options = dict(options or {})
    crossover = bool(options.pop("crossover", False))
    key = (family, mode, T, n_tracking_hour, tuple(sorted(options.items())))
    if key not in _SOLVERS:
        _SOLVERS[key] = BatchLPSolver(_FAMILIES[family](T, mode, n_tracking_hour), **options)
    sol = _SOLVERS[key]
    if not crossover:
        r = sol.solve_host(np.ascontiguousarray(cparams), np.ascontiguousarray(rparams), want_x=True)
        return r.obj, r.status, _columns(sol.t, sol.to_model_space(r.x), T)
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    cp = torch.as_tensor(np.ascontiguousarray(cparams, float), device=dev)
    rp = torch.as_tensor(np.ascontiguousarray(rparams, float), device=dev)
    r = sol.solve(cp, rp, want_x=True, want_y=True)
    v = sol.crossover(cp, rp, r)
    ok = (v.status == OPTIMAL)
    x = torch.where(ok[:, None], v.x, r.x).cpu().numpy()
    obj = torch.where(ok, v.obj, r.obj).cpu().numpy()
    return obj, r.status.cpu().numpy(), _columns(sol.t, sol.to_model_space(x), T)


_COLS = dict(grid="blk[{t}].fs.splitter.grid_elec[0]", batt_in="blk[{t}].fs.battery.elec_in[0]",
             batt_out="blk[{t}].fs.battery.elec_out[0]", soc="blk[{t}].fs.battery.state_of_charge[0]",
             throughput="blk[{t}].fs.battery.energy_throughput[0]", waste="wind_waste_kw[{t}]",
             under="power_underdelivered_kw[{t}]", over="power_overdelivered_kw[{t}]",
             da="day_ahead_power_kw[{t}]", underbid="real_time_underbid_power_kw[{t}]",
             pem="blk[{t}].fs.pem.electricity[0]", pipeline="blk[{t}].fs.h2_tank.outlet_to_pipeline.flow_mol[0]",
             holdup="blk[{t}].fs.h2_tank.tank_holdup[0]", pem_cap="pem_system_capacity[{t}]")


def _columns(template, xm, T):
    cn = {n: j for j, n in enumerate(template.col_names)}
    out = {}
    for k, pat in _COLS.items():
        if pat.format(t=0) in cn:
            out[k] = xm[:, [cn[pat.format(t=t)] for t in range(T)]]
    return out


def _result_frame(N, H, const_cols, array_cols, kwargs):
    """The reference builds its result table row by row; here one frame per call from [N, H] arrays (rounded to 2
    decimals like the reference), row order (simulation, horizon hour)."""
    import pandas as pd
    data = {k: [v] * (N * H) for k, v in const_cols.items()}
    data["Horizon [hr]"] = np.tile(np.arange(H), N)
    for k, a in array_cols.items():
        data[k] = np.round(np.asarray(a, float).reshape(N * H), 2)
    if N > 1:
        data["Simulation"] = np.repeat(np.arange(N), H)
    for k, v in kwargs.items():
        data[k] = [v] * (N * H)
    return pd.DataFrame(data)


# ---- minimal stand-ins for idaes.apps.grid_integration.model_data (only the fields the reference's tests set)
@dataclasses.dataclass
class RenewableGeneratorModelData:
    gen_name: str
    bus: str
    p_min: float
    p_max: float
    p_cost: float = 0.0
    fixed_commitment: object = None
    generator_type = "renewable"


@dataclasses.dataclass
class ThermalGeneratorModelData:
    gen_name: str
    bus: str
    p_min: float
    p_max: float
    min_down_time: float = 0
    min_up_time: float = 0
    ramp_up_60min: float = 0
    ramp_down_60min: float = 0
    shutdown_capacity: float = 0
    startup_capacity: float = 0
    initial_status: int = 1
    initial_p_output: float = 0
    production_cost_bid_pairs: list = None
    include_default_p_cost: bool = False
    startup_cost_pairs: list = None
    fixed_commitment: object = None
    generator_type = "thermal"


class Backcaster:
    """Price forecaster: scenario k replays the historical days in reverse chronological order starting k days back
    (pinned by the reference's 48-h known bids for k = 0, test_multiperiod_wind_battery_doubleloop.py:124-129,168-175)."""

    def __init__(self, historical_da_prices, historical_rt_prices, max_historical_days=10):
        self._da = {b: list(np.asarray(v, float)) for b, v in historical_da_prices.items()}
        self._rt = {b: list(np.asarray(v, float)) for b, v in historical_rt_prices.items()}
        for hist in (self._da, self._rt):
            for b, v in hist.items():
                if len(v) < 24:
                    raise ValueError(f"At least a day of the historical prices for bus {b} is required.")
        self.max_historical_days = max_historical_days

    @staticmethod
    def _forecast(hist, hour, horizon, n_samples):
        h = np.asarray(hist, float)
        days = h[: (h.size // 24) * 24].reshape(-1, 24)
        nd = days.shape[0]
        reps = (hour + horizon) // 24 + 1
        return np.array([np.concatenate([days[(nd - 1 - k - r) % nd] for r in range(reps)])[hour:hour + horizon]
                         for k in range(n_samples)])

    def forecast_day_ahead_prices(self, date, hour, bus, horizon, n_samples):
        return self._forecast(self._da[bus], hour, horizon, n_samples)

    def forecast_real_time_prices(self, date, hour, bus, horizon, n_samples):
        return self._forecast(self._rt[bus], hour, horizon, n_samples)

    def forecast_day_ahead_and_real_time_prices(self, date, hour, bus, horizon, n_samples):
        return (self.forecast_day_ahead_prices(date, hour, bus, horizon, n_samples),
                self.forecast_real_time_prices(date, hour, bus, horizon, n_samples))

    def fetch_hourly_stats_from_prescient(self, *a, **k):       # bookkeeping hook of the co-simulation; nothing to solve
        raise NotImplementedError("Prescient co-simulation is outside the hot path (SURVEY.md §8)")


class _Block:
    """What ``populate_model`` fills: the state the reference keeps on a Pyomo block (sizes live on the model object)."""
    def __init__(self):
        self.horizon = 0
        self._time_idx = 0
        self.soc0 = None            # [N] kWh
        self.thr0 = None            # [N] kWh
        self.cf = None              # [N, horizon]
        self.wind_waste_penalty = 1e3          # wind_battery_double_loop.py:165
        self.sol = None             # columns of the last solve, kW / kWh, each [N, horizon]
        self.P_T = None             # [N, horizon] MW
        self.tot_cost = None        # [N, horizon] $
        self.wind_waste = None      # [N, horizon] MW


class MultiPeriodWindBattery:
    """wind_battery_double_loop.py:104-352.  ``wind_capacity_factors`` [L] or [N, L]; sizes scalar or [N]."""

    def __init__(self, model_data, wind_capacity_factors=None, wind_pmax_mw=200.0, battery_pmax_mw=25.0,
                 battery_energy_capacity_mwh=100.0):
        self.model_data = model_data
        if wind_capacity_factors is None:
            raise ValueError("Please provide wind capacity factors.")       # :130-131
        self._wind_capacity_factors = np.atleast_2d(np.asarray(wind_capacity_factors, float))
        N = self._wind_capacity_factors.shape[0]
        sizes = np.broadcast_arrays(np.zeros(N), wind_pmax_mw, battery_pmax_mw, battery_energy_capacity_mwh)
        self.N = sizes[0].shape[0]
        if N == 1 and self.N > 1:
            self._wind_capacity_factors = np.repeat(self._wind_capacity_factors, self.N, axis=0)
        self._wind_pmax_mw, self._battery_pmax_mw, self._battery_energy_capacity_mwh = (np.array(s, float) for s in sizes[1:])
        self.result_list = []

    # -- populate / update (:141-206)
    def populate_model(self, b, horizon):
        b.horizon = horizon
        b._time_idx = 0
        b.soc0 = np.zeros(self.N)          # initial_state_of_charge fixed at its initial value 0 (:76-77)
        b.thr0 = np.zeros(self.N)          # initial_energy_throughput: free until the first update; 0 is optimal
        b.cf = self._wind_capacity_factors[:, 0:horizon].copy()
        return b

    def update_model(self, b, realized_soc, realized_energy_throughput):
        """realized_* : sequences (deque) of per-hour values, each a scalar or [N] (kWh)."""
        b.soc0 = np.round(np.broadcast_to(np.asarray(realized_soc[-1], float), (self.N,)), 2)               # :189-191
        b.thr0 = np.round(np.broadcast_to(np.asarray(realized_energy_throughput[-1], float), (self.N,)), 2)  # :193-196
        b._time_idx = b._time_idx + min(len(realized_soc), 24)                                                # :199-200
        b.cf = self._get_capacity_factors(b)

    def _get_capacity_factors(self, b):
        L = self._wind_capacity_factors.shape[1]
        ans = self._wind_capacity_factors[:, b._time_idx:b._time_idx + b.horizon]
        if ans.shape[1] < b.horizon:                                                                          # :222-223
            ans = np.concatenate([ans, self._wind_capacity_factors[:, 0:b.horizon - ans.shape[1]]], axis=1)
        return ans

    # -- rparams / post-processing shared by the tracker and the bidders
    def _rparams(self, b, signal_mw=None):
        return TP.wind_battery_operation_rparams(b.horizon, b.cf, self._wind_pmax_mw, self._battery_pmax_mw,
                                                 self._battery_energy_capacity_mwh, b.soc0, b.thr0, signal_mw)

    def _lp(self, b, mode, da=None, rt=None, signal_mw=None, n_tracking_hour=1, options=None):
        """Solves the block's LP in the given mode for all N simulations and loads the solution into the block."""
        pen = np.full((self.N, 1), b.wind_waste_penalty)
        cp = pen if mode == "tracker" else np.concatenate([da, rt, pen], axis=1)
        obj, status, cols = _lp_solve(mode, b.horizon, cp, self._rparams(b, signal_mw), n_tracking_hour, options, "wind_battery")
        self._load_solution(b, cols)
        return obj, status, cols

    def _load_solution(self, b, cols):
        b.sol = cols
        b.P_T = (cols["grid"] + cols["batt_out"]) * 1e-3                                                      # :168
        b.wind_waste = cols["waste"] * 1e-3                                                                   # :169
        prev = np.concatenate([b.thr0[:, None], cols["throughput"][:, :-1]], axis=1)
        kdeg = TP.DEGRADATION * TP.BATT_REP_COST_KWH
        b.tot_cost = (self._wind_pmax_mw[:, None] * 1e3 * TP.WIND_OP_COST / 8760.0 + kdeg * (cols["throughput"] - prev)
                      + b.wind_waste_penalty * b.wind_waste)                                                  # :170-171

    @staticmethod
    def get_last_delivered_power(b, last_implemented_time_step):
        return b.P_T[:, last_implemented_time_step]                                                           # :239-240

    @staticmethod
    def get_implemented_profile(b, last_implemented_time_step):
        n = last_implemented_time_step + 1
        return {"realized_soc": deque(b.sol["soc"][:, t] for t in range(n)),                                  # :257-270
                "realized_energy_throughput": deque(b.sol["throughput"][:, t] for t in range(n))}

    def record_results(self, b, date=None, hour=None, **kwargs):
        """Rows of the reference's result table (:272-335), one per (simulation, horizon hour)."""
        H = b.horizon
        cols = {"Total Wind Generation [MW]": (b.sol["grid"] + b.sol["batt_in"]) * 1e-3,
                "Total Power Output [MW]": b.P_T,
                "Wind Power Output [MW]": b.sol["grid"] * 1e-3,
                "Wind Curtailment [MW]": np.repeat(b.wind_waste[:, :1], H, axis=1),        # the reference reads index 0 (:309)
                "Battery Power Output [MW]": b.sol["batt_out"] * 1e-3,
                "Wind Power to Battery [MW]": b.sol["batt_in"] * 1e-3,
                "State of Charge [MWh]": b.sol["soc"] * 1e-3,
                "Total Cost [$]": b.tot_cost}
        self.result_list.append(_result_frame(self.N, H, {"Generator": self.model_data.gen_name, "Date": date, "Hour": hour},
                                              cols, kwargs))

    def write_results(self, path):
        import pandas as pd
        pd.concat(self.result_list).to_csv(path, index=False)                                                  # :344

    @property
    def power_output(self):
        return "P_T"

    @property
    def total_cost(self):
        return ("tot_cost", 1)


class MultiPeriodWindPEM:
    """wind_PEM_double_loop.py:103-330 (wind + PEM, battery size 0).  Only the Tracker solves an LP with this model; the
    reference's bidder for it (PEM_parametrized_bidder.py) derives its bids from forecasts without optimisation."""

    def __init__(self, model_data, wind_capacity_factors, wind_pmax_mw=200.0, pem_pmax_mw=25.0):
        self.model_data = model_data
        if wind_capacity_factors is None:
            raise ValueError("Please provide wind capacity factors.")                                       # :125-126
        self._wind_capacity_factors = np.atleast_2d(np.asarray(wind_capacity_factors, float))
        N = self._wind_capacity_factors.shape[0]
        sizes = np.broadcast_arrays(np.zeros(N), wind_pmax_mw, pem_pmax_mw)
        self.N = sizes[0].shape[0]
        if N == 1 and self.N > 1:
            self._wind_capacity_factors = np.repeat(self._wind_capacity_factors, self.N, axis=0)
        self._wind_pmax_mw, self._pem_pmax_mw = (np.array(x, float) for x in sizes[1:])
        self.result_list = []

    def populate_model(self, b, horizon):
        b.horizon, b._time_idx = horizon, 0
        b.cf = self._wind_capacity_factors[:, 0:horizon].copy()
        return b

    def update_model(self, b, realized_h2_sales):
        b._time_idx = b._time_idx + min(len(realized_h2_sales), 24)                                         # :196-197
        b.cf = self._get_capacity_factors(b)

    def _get_capacity_factors(self, b):
        ans = self._wind_capacity_factors[:, b._time_idx:b._time_idx + b.horizon]
        if ans.shape[1] < b.horizon:                                                                         # :219-220
            ans = np.concatenate([ans, self._wind_capacity_factors[:, 0:b.horizon - ans.shape[1]]], axis=1)
        return ans

    def _lp(self, b, mode, da=None, rt=None, signal_mw=None, n_tracking_hour=1, options=None):
        if mode != "tracker":
            raise NotImplementedError("MultiPeriodWindPEM is bid with the parametrised bidder (no LP); only the Tracker solves one")
        T = b.horizon
        W = self._wind_pmax_mw[:, None] * 1e3
        sig = np.broadcast_to(np.atleast_2d(np.asarray(signal_mw, float)), (self.N, T))
        rp = np.concatenate([b.cf * W, W, sig], axis=1)
        obj, status, cols = _lp_solve(mode, T, np.ones((self.N, 1)), rp, n_tracking_hour, options, "wind_pem")
        b.sol = cols
        b.P_T = cols["grid"] * 1e-3                                                                          # :168
        b.wind_waste = cols["waste"]                                                                         # :169 (kW)
        b.tot_cost = (W * TP.WIND_OP_COST / 8760.0 + cols["pem_cap"] * TP.PEM_OP_COST / 8760.0
                      + TP.PEM_VAR_COST * cols["pem"] + b.wind_waste)                                        # :170-172
        return obj, status, cols

    @staticmethod
    def get_last_delivered_power(b, last_implemented_time_step):
        return b.P_T[:, last_implemented_time_step]

    @staticmethod
    def get_implemented_profile(b, last_implemented_time_step):
        k = TP.PEM_ELEC_TO_MOL / TP.H2_MOLS_PER_KG * 3600.0
        return {"realized_h2_sales": deque(b.sol["pem"][:, t] * k for t in range(last_implemented_time_step + 1))}   # :253-256

    def record_results(self, b, date=None, hour=None, **kwargs):
        """Rows of the reference's table (:265-320)."""
        k = TP.PEM_ELEC_TO_MOL / TP.H2_MOLS_PER_KG * 3600.0
        H = b.horizon
        cols = {"Total Wind Generation [MW]": (b.sol["grid"] + b.sol["pem"]) * 1e-3,
                "Total Power Output [MW]": b.P_T,
                "Wind Power Output [MW]": b.sol["grid"] * 1e-3,
                "Wind to PEM [MW]": b.sol["pem"] * 1e-3,
                "Wind Curtailment [MW]": np.repeat(b.wind_waste[:, :1], H, axis=1),        # the reference reads index 0, in kW (:302)
                "Hydrogen Sales [kg]": b.sol["pem"] * k,
                "Total Cost [$]": b.tot_cost}
        self.result_list.append(_result_frame(self.N, H, {"Generator": self.model_data.gen_name, "Date": date, "Hour": hour},
                                              cols, kwargs))

    def write_results(self, path):
        import pandas as pd
        pd.concat(self.result_list).to_csv(path, index=False)

    @property
    def power_output(self):
        return "P_T"

    @property
    def total_cost(self):
        return ("tot_cost", 1)


class MultiPeriodNuclear:
    """nuclear_flowsheet_multiperiod_class.py:158-344 (500 MW NPP + 100 MW PEM + 5000 kg tank, :97-102).  ``n_sim``
    independent simulations share the plant data and differ in their market signals / implemented hold-ups."""
    MW_H2 = 2.016e-3

    def __init__(self, model_data, n_sim=1, h2_price=4.0):
        self.model_data = model_data
        self.p_lower, self.p_upper, self.generator = model_data.p_min, model_data.p_max, model_data.gen_name   # :181-183
        self.N, self.h2_price = int(n_sim), h2_price
        self.result_list = []

    def populate_model(self, blk, horizon):
        blk.horizon = horizon
        blk.holdup0 = np.zeros(self.N)                              # tank_holdup_previous of block 0 fixed to 0 (:203)
        return blk

    def update_model(self, b, implemented_tank_holdup):
        b.holdup0 = np.round(np.broadcast_to(np.asarray(implemented_tank_holdup[-1], float), (self.N,)))   # :232-235

    def _lp(self, b, mode, da=None, rt=None, signal_mw=None, n_tracking_hour=1, options=None):
        T = b.horizon
        h2 = np.full((self.N, 1), self.h2_price)
        cp = h2 if mode == "tracker" else np.concatenate([da, rt, h2], axis=1)
        sig = np.zeros((self.N, T)) if signal_mw is None else np.broadcast_to(np.atleast_2d(np.asarray(signal_mw, float)), (self.N, T))
        rp = np.concatenate([b.holdup0[:, None], sig], axis=1)
        obj, status, cols = _lp_solve(mode, T, cp, rp, n_tracking_hour, options, "nuclear")
        E = TP.NUC_NP_CAPACITY_MW * 1e3
        b.sol = cols
        b.P_T = (E - cols["pem"]) * 1e-3                                                             # :211
        b.tot_cost = (E * 1e-3 * 2.3 + cols["pem"] * 1e-3 * 1.3 + cols["holdup"] * self.MW_H2 * 0.01
                      - cols["pipeline"] * self.MW_H2 * 3600.0 * self.h2_price)                      # :149-153, :212
        return obj, status, cols

    @staticmethod
    def get_last_delivered_power(b, last_implemented_time_step):
        return b.P_T[:, last_implemented_time_step]                                                  # :252

    @staticmethod
    def get_implemented_profile(b, last_implemented_time_step):
        return {"implemented_tank_holdup": deque(b.sol["holdup"][:, t] for t in range(last_implemented_time_step + 1))}

    def record_results(self, blk, date=None, hour=None, **kwargs):
        """Rows of the reference's table (:281-320)."""
        prev = np.concatenate([blk.holdup0[:, None], blk.sol["holdup"][:, :-1]], axis=1)
        cols = {"Power to Grid [MW]": blk.P_T,
                "Power to PEM [MW]": blk.sol["pem"] * 1e-3,
                "Initial holdup [kg]": prev * self.MW_H2,
                "Final holdup [kg]": blk.sol["holdup"] * self.MW_H2,
                "Hydrogen Market [kg/hr]": blk.sol["pipeline"] * self.MW_H2 * 3600,
                "Total Cost [$]": blk.tot_cost}
        self.result_list.append(_result_frame(self.N, blk.horizon, {"Date": date, "Hour": hour}, cols, kwargs))

    def write_results(self, path):
        import pandas as pd
        pd.concat(self.result_list).to_csv(path, index=False)

    @property
    def power_output(self):
        return "P_T"

    @property
    def total_cost(self):
        return ("tot_cost", 1)

    @property
    def pmin(self):
        return self.p_lower


class Tracker:
    """idaes Tracker as the reference drives it (test_multiperiod_wind_battery_doubleloop.py:68-87): one LP per call of
    ``track_market_dispatch`` over ``tracking_horizon`` hours, the first ``n_tracking_hour`` tracked hard."""

    def __init__(self, tracking_model_object, tracking_horizon, n_tracking_hour, solver=None):
        self.tracking_model_object = tracking_model_object
        self.tracking_horizon, self.n_tracking_hour = int(tracking_horizon), int(n_tracking_hour)
        self.solver_options = dict(solver or {})
        self.fs = _Block()
        tracking_model_object.populate_model(self.fs, self.tracking_horizon)
        self.daily_stats, self.projection, self.result_list = None, None, []
        self.status = None

    @property
    def power_output(self):
        return self.fs.P_T

    def track_market_dispatch(self, market_dispatch, date, hour):
        obj_ = self.tracking_model_object
        N, H = obj_.N, self.tracking_horizon
        md = np.broadcast_to(np.atleast_2d(np.asarray(market_dispatch, float)), (N, H))
        obj, status, cols = obj_._lp(self.fs, "tracker", signal_mw=md, n_tracking_hour=self.n_tracking_hour,
                                     options=self.solver_options)
        self.status = status
        if np.any(status != OPTIMAL):
            raise RuntimeError(f"tracking LP not optimal for simulations {np.nonzero(status != OPTIMAL)[0][:8].tolist()}")
        self.objective = obj
        self.power_underdelivered, self.power_overdelivered = cols["under"] * 1e-3, cols["over"] * 1e-3
        obj_.record_results(self.fs, date=date, hour=hour)
        last = self.n_tracking_hour - 1
        profiles = obj_.get_implemented_profile(self.fs, last)
        self._last_delivered = obj_.get_last_delivered_power(self.fs, last).copy()
        obj_.update_model(self.fs, **profiles)
        return profiles

    def get_last_delivered_power(self):
        return self._last_delivered


class _StochasticProgramBidder:
    def __init__(self, bidding_model_object, day_ahead_horizon, real_time_horizon, n_scenario, solver=None, forecaster=None):
        if n_scenario != 1:
            raise NotImplementedError("n_scenario > 1 couples the scenario blocks (non-anticipativity rows): not batched yet")
        self.bidding_model_object = bidding_model_object
        self.day_ahead_horizon, self.real_time_horizon = int(day_ahead_horizon), int(real_time_horizon)
        self.n_scenario, self.forecaster = n_scenario, forecaster
        self.solver_options = dict(solver or {})
        self.generator = bidding_model_object.model_data.gen_name
        self.day_ahead_model, self.real_time_model = _Block(), _Block()
        bidding_model_object.populate_model(self.day_ahead_model, self.day_ahead_horizon)
        bidding_model_object.populate_model(self.real_time_model, self.real_time_horizon)
        self.bids_result_list = []

    def _forecasts(self, which, date, hour, horizon):
        """[N, horizon] forecast prices; a forecaster per simulation may be given as a list."""
        N = self.bidding_model_object.N
        fcs = self.forecaster if isinstance(self.forecaster, (list, tuple)) else [self.forecaster] * N
        bus = self.bidding_model_object.model_data.bus
        out = np.array([getattr(f, which)(date=date, hour=hour, bus=bus, horizon=horizon, n_samples=1)[0] for f in fcs])
        return out

    def _solve(self, blk, mode, da, rt, da_dispatch=None):
        obj_ = self.bidding_model_object
        N, H = obj_.N, blk.horizon
        obj, status, cols = obj_._lp(blk, mode, da=da, rt=rt, signal_mw=da_dispatch, options=self.solver_options)
        if np.any(status != OPTIMAL):
            raise RuntimeError(f"bidding LP not optimal for simulations {np.nonzero(status != OPTIMAL)[0][:8].tolist()}")
        if da_dispatch is not None:                      # constant dropped from the template (bilinear in the parameters)
            obj = obj - np.sum((da - rt) * da_dispatch, axis=1)
        blk.objective = -obj                             # the IDAES objective is a maximisation
        return cols

    def compute_day_ahead_bids(self, date, hour=0):
        H = self.day_ahead_horizon
        da = self._forecasts("forecast_day_ahead_prices", date, hour, H)
        rt = self._forecasts("forecast_real_time_prices", date, hour, H)
        cols = self._solve(self.day_ahead_model, "bidder_da", da, rt)
        self.day_ahead_power = cols["da"] * 1e-3                       # [N, H] MW
        bids = self._assemble_bids(self.day_ahead_power, da, hour)
        self.bidding_model_object.record_results(self.day_ahead_model, date=date, hour=hour, market="Day-ahead")
        return bids

    def compute_real_time_bids(self, date, hour, realized_day_ahead_prices, realized_day_ahead_dispatches):
        H = self.real_time_horizon
        N = self.bidding_model_object.N

        def window(a):                                                  # hours past the end repeat the last value
            a = np.broadcast_to(np.atleast_2d(np.asarray(a, float)), (N, np.shape(a)[-1]))
            idx = np.minimum(np.arange(hour, hour + H), a.shape[1] - 1)
            return a[:, idx]
        da, disp = window(realized_day_ahead_prices), window(realized_day_ahead_dispatches)
        rt = self._forecasts("forecast_real_time_prices", date, hour, H)
        cols = self._solve(self.real_time_model, "bidder_rt", da, rt, disp)
        self.real_time_underbid_power = cols["underbid"] * 1e-3
        bids = self._assemble_bids(self.real_time_model.P_T, rt, hour)
        self.bidding_model_object.record_results(self.real_time_model, date=date, hour=hour, market="Real-time")
        return bids

    def update_day_ahead_model(self, **profiles):
        self.bidding_model_object.update_model(self.day_ahead_model, **profiles)

    def update_real_time_model(self, **profiles):
        self.bidding_model_object.update_model(self.real_time_model, **profiles)

    @staticmethod
    def _scalar(a):
        a = np.asarray(a)
        return float(a[0]) if a.size == 1 else a


class SelfScheduler(_StochasticProgramBidder):
    """Self-schedule bids: p_max[t] = the scheduled power, rounded to 4 decimals
    (the reference reads ``bids[t][gen]['p_max']``, test_multiperiod_wind_battery_doubleloop.py:154-156)."""

    def _assemble_bids(self, power_mw, prices, hour):
        md = self.bidding_model_object.model_data
        bids = {}
        for t in range(power_mw.shape[1]):
            p = np.round(power_mw[:, t], 4)
            bids[t + hour] = {self.generator: {"p_min": md.p_min, "p_max": self._scalar(p), "p_min_agc": md.p_min,
                                               "p_max_agc": self._scalar(p), "p_cost": getattr(md, "p_cost", 0.0)}}
        return bids


class Bidder(_StochasticProgramBidder):
    """Price-quantity bids of a thermal-type participant: per hour the curve [(p_min, 0), (P, P*price)] built from the
    scenario's (power, price) pair (the reference reads ``bids[t][gen]['p_cost'][-1][1]``, :233-236)."""

    def _assemble_bids(self, power_mw, prices, hour):
        md = self.bidding_model_object.model_data
        bids = {}
        for t in range(power_mw.shape[1]):
            p = np.round(np.maximum(power_mw[:, t], md.p_min), 4)
            cost = np.round(np.round(prices[:, t], 4) * (p - md.p_min), 4)
            curve = [(md.p_min, 0.0), (self._scalar(p), self._scalar(cost))]
            bids[t + hour] = {self.generator: {"p_cost": curve, "p_min": md.p_min, "p_max": self._scalar(p),
                                               "startup_capacity": md.p_min, "shutdown_capacity": md.p_min}}
        return bids
