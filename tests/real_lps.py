"""Real, degenerate dispatch LPs with certified exact optima (test infrastructure, no GPU).

The LPs the project solves are primal and dual degenerate: a quarter of the hours have a zero price, batteries sit empty and
idle, capacity factors are 0.  Their x and y are then not unique, and the planted generators (planted_stage.py) cannot stand in
for them.  Each set here is built deterministically from the committed price / capacity-factor pool (dispatches_b200/data) and
the scenario batches of dispatches_b200/scenarios.py, certified LP by LP with exact_lp.exact_optimum (HiGHS' final basis,
verified in exact arithmetic, or its exact repair) and cached per process.  The sets cover the wind + battery dispatch (C2, C5,
real windows of 2 to 256 hours, the edges), nuclear, fossil, wind + battery + PEM, the double-loop operation LPs, battery design,
and PV + battery + hydrogen at fixed sizes and in design (one PV series baked into A, or one per LP as matrix coefficients) over
24 hours to a week (m = 363 to 2 523; a week-long design LP takes about 70 s on one core, so the long sets take ``procs``).  Not
covered: the free-wind design, which HiGHS reports unbounded at 1e-10 tolerances, and the full-year LPs, whose exact certification
would take far longer.

``check_exact`` measures a kernel's answer on such a set against what every optimum of the LP shares: the objective, the KKT
conditions, x / y element-wise where they are unique, and on every LP the columns every optimal x has at a bound (``fixed``)
and the columns at which every optimal y has a zero reduced cost (``inside``).
"""
from __future__ import annotations

import dataclasses
import functools
import json
import multiprocessing as mp
from pathlib import Path

import numpy as np

from dispatches_b200 import scenarios as SC
from dispatches_b200 import templates as TP
from dispatches_b200.lp_template import LPTemplate
from exact_lp import exact_optimum, kkt_residuals
from planted_lp import rel
from planted_stage import KKT_DUAL, KKT_GAP, KKT_PRIMAL, OBJ_REL, XY_REL

# The two margins of the element-wise checks on degenerate LPs.  An interior-point iterate stops with x_j ~ mu / r_j on a column
# with reduced cost r_j, and with r_j(y) ~ mu / x_j on a column at x_j: a column whose exact reduced cost is far below |c|_inf
# (or whose x*_j is far below |x*|_inf) is legitimately not at its limit yet.  The planted suite keeps r_margin >= 1e-3 and
# x_margin >= 1e-2 for the same reason.
R_MARGIN = 1e-3      # `fixed` columns checked: |r*_j| >= R_MARGIN |c|_inf
X_MARGIN = 1e-2      # `inside` columns checked: x*_j at least X_MARGIN max(1, |x*|_inf) from both bounds


@dataclasses.dataclass
class ExactSet:
    t: LPTemplate
    cparams: np.ndarray        # [N, Pc]
    rparams: np.ndarray        # [N, Pr] (Pr may be 0)
    x: np.ndarray              # [N, n] an exact optimum, template column order
    y: np.ndarray              # [N, m] its exact row duals
    r: np.ndarray              # [N, n] exact reduced costs c - A'y*
    obj: np.ndarray            # [N] c'x* + k
    lp_mag: np.ndarray         # [N] sum_j |c_j x*_j|
    fixed: np.ndarray          # [N, n] bool
    inside: np.ndarray         # [N, n] bool
    unique_x: np.ndarray       # [N] bool
    unique_y: np.ndarray       # [N] bool
    u: np.ndarray              # [N, n] the instantiated upper bounds (inf where none)
    csc: np.ndarray            # [N] |c|_inf
    x_margin: np.ndarray       # [N] ExactOptimum.x_margin
    r_margin: np.ndarray       # [N] ExactOptimum.r_margin
    pivots: np.ndarray         # [N] ExactOptimum.pivots: exact dual simplex pivots that repaired HiGHS' basis
    col: np.ndarray            # [N, n] int8 and
    row_basic: np.ndarray      # [N, m] bool: the verified basis of each LP (ExactOptimum.basis)

    def __len__(self):
        return len(self.obj)

    def take(self, k):
        return dataclasses.replace(self, **{f.name: getattr(self, f.name)[k] for f in dataclasses.fields(self) if f.name != "t"})

    def tile(self, N, seed=0):
        """N LPs: the set repeated in a random permutation (every copy bitwise equal to its first copy)"""
        k = np.random.default_rng(seed).permutation(np.resize(np.arange(len(self)), N))
        return self.take(k), k


def _certify_one(args):
    t, cp, rp = args
    e = exact_optimum(t, cp, rp)
    c, _, u, _ = t.instantiate(cp, rp)
    return e, u, float(np.abs(c).max(initial=0.0))


def certify(t, cparams, rparams, procs=1):
    """the exact optimum of every LP (raises exact_lp.NotCertified on the first that does not certify)"""
    cparams = np.ascontiguousarray(np.atleast_2d(cparams), float)
    N = len(cparams)
    rparams = np.zeros((N, 0)) if rparams is None else np.ascontiguousarray(np.broadcast_to(rparams, (N, np.shape(rparams)[-1])), float)
    jobs = [(t, cparams[k], rparams[k]) for k in range(N)]
    if procs > 1 and N > 1:
        with mp.get_context("fork").Pool(min(procs, N)) as pool:
            out = pool.map(_certify_one, jobs, chunksize=max(1, N // (4 * procs)))
    else:
        out = [_certify_one(j) for j in jobs]
    es = [o[0] for o in out]
    st = lambda f: np.array([getattr(e, f) for e in es])
    return ExactSet(t, cparams, rparams, st("x"), st("y"), st("r"), st("obj"), st("lp_mag"), st("fixed"), st("inside"),
                    st("unique_x"), st("unique_y"), np.array([o[1] for o in out]), np.array([o[2] for o in out]), st("x_margin"),
                    st("r_margin"), st("pivots"), np.array([e.basis[0] for e in es]), np.array([e.basis[1] for e in es]))


# ---------------------------------------------------------------------------------------------------------------------
# LP sets (deterministic; cached per process)
# ---------------------------------------------------------------------------------------------------------------------
def _wb(T, lmp, cf, wind_mw, batt_mw):
    return certify(TP.wind_battery(T), lmp, TP.wind_battery_rparams(T, cf, wind_mw, batt_mw))


@functools.lru_cache(maxsize=None)
def c2(N=64, stride=None):
    """LPs 0, s, 2 s, ... of the headline batch scenarios.c2() (10 000 LPs, T = 24); s = 10 000 // N by default"""
    lmp, cf, W, P = SC.c2()
    k = np.arange(N) * (stride or len(lmp) // N)
    return _wb(24, lmp[k], cf, W, P)


C5_STRIDE = 2803         # 201 of the 560 640 design-sweep LPs: every wind size and battery ratio, start hours spread over the year


@functools.lru_cache(maxsize=None)
def c5(N=None, stride=C5_STRIDE):
    lmp, cf, W, P = SC.c5()
    k = np.arange(0, len(lmp), stride)[:N]
    return _wb(24, lmp[k], cf[k], W[k], P[k])


@functools.lru_cache(maxsize=None)
def windows(T, N=16, seed=0):
    """real T-hour windows of the 303 day-ahead price and wind series at seeded start hours, W = 847 MW, battery 0.25 W"""
    p = SC.pool()
    h0 = np.random.default_rng([T, seed]).integers(0, len(p["dalmp_303"]) - T, N)
    idx = h0[:, None] + np.arange(T)[None, :]
    return _wb(T, p["dalmp_303"][idx], p["dacf_303"][idx], SC.FIXED_WIND_MW, 0.25 * SC.FIXED_WIND_MW)


EDGES = ("zero_prices", "negative_prices", "spike", "whole_dollars", "zero_cf", "no_battery", "small_battery")


@functools.lru_cache(maxsize=None)
def edges(per_case=4):
    """the real edges of the 24-hour dispatch LP, ``per_case`` LPs each, in EDGES order: all-zero prices; negative prices (the
    real day windows with hours below 0); one 10 000 $/MWh spike in an otherwise real day; prices rounded to whole dollars (many
    ties); days with three or more zero capacity-factor hours; battery P = 0 (every battery column fixed at 0); 5 % batteries (the
    smallest ratio of C5).  Wind 847 MW, battery 0.25 x that unless the case says otherwise."""
    T = 24
    p = SC.pool()
    lam, cf = p["dalmp_303"], p["dacf_303"]
    days = np.arange(len(lam) // T) * T
    rng = np.random.default_rng(7)
    neg = p["day_windows"][(p["day_windows"] < 0).any(1)]
    zero_cf = days[np.array([(cf[h:h + T] == 0).sum() >= 3 for h in days])]
    W = SC.FIXED_WIND_MW
    lmps, cfs, batt = [], [], []
    for case in EDGES:
        h = np.sort(rng.choice(zero_cf if case == "zero_cf" else days, per_case, replace=False))
        idx = h[:, None] + np.arange(T)[None, :]
        lm, c = lam[idx].copy(), cf[idx].copy()
        b = np.full(per_case, 0.25 * W)
        if case == "zero_prices":
            lm[:] = 0.0
        elif case == "negative_prices":
            lm = neg[rng.choice(len(neg), per_case, replace=len(neg) < per_case)]
        elif case == "spike":
            lm[np.arange(per_case), rng.integers(0, T, per_case)] = 10000.0
        elif case == "whole_dollars":
            lm = np.round(lm)
        elif case == "no_battery":
            b[:] = 0.0
        elif case == "small_battery":
            b[:] = 0.05 * W
        lmps.append(lm); cfs.append(c); batt.append(b)
    return _wb(T, np.concatenate(lmps), np.concatenate(cfs), W, np.concatenate(batt))


def edge_rows(name, per_case=4):
    i = EDGES.index(name)
    return np.arange(i * per_case, (i + 1) * per_case)


@functools.lru_cache(maxsize=None)
def nuclear(T, N=16):
    """nuclear(T) on consecutive real cluster days (scenarios.c3 draws, truncated or extended to T hours)"""
    p = SC.pool()["cluster_days"]
    rng = np.random.default_rng([T, 3])
    d = rng.integers(0, len(p) - 5, N)
    lmp = np.stack([np.concatenate([p[k + i] for i in range(5)])[:T] for k in d]) * rng.lognormal(0, 0.25, (N, T))
    return certify(TP.nuclear(T), lmp, None)


@functools.lru_cache(maxsize=None)
def nuclear_report(T, N=16):
    """nuclear_report(T) on real-time report prices, with hydrogen price and the three capacities varied per LP"""
    lam = SC.pool()["nuc_report_lmp_rt"]
    rng = np.random.default_rng([T, 4])
    h0 = rng.integers(0, len(lam) - T, N)
    cp = np.concatenate([lam[h0[:, None] + np.arange(T)[None, :]], rng.uniform(0.75, 3.0, (N, 1))], axis=1)
    rp = np.stack([rng.uniform(20.0, 200.0, N), rng.uniform(0.0, 50000.0, N), rng.uniform(0.0, 40.0, N)], axis=1)
    return certify(TP.nuclear_report(T), cp, rp)


@functools.lru_cache(maxsize=None)
def fossil(T=168, N=8):
    return certify(TP.fossil_surrogate(T), SC.c4(N), None)


@functools.lru_cache(maxsize=None)
def wind_battery_pem(T=24, with_battery=True, N=16):
    lmp, cf, W, P = SC.c2(N, seed=5)
    cp = np.concatenate([lmp, np.full((N, 1), 2.5)], axis=1)
    rp = TP.wind_battery_rparams(T, cf, W, 150.0 if with_battery else 0.0, pem_mw=200.0)
    return certify(TP.wind_battery_pem(T, with_battery=with_battery), cp, rp)


OPERATIONS = ("wind_battery_tracker", "wind_battery_bidder_da", "nuclear_tracker", "nuclear_bidder_da", "wind_pem_tracker")


@functools.lru_cache(maxsize=None)
def operation(name, T=24, N=8):
    """the double-loop tracker and day-ahead bidder LPs on real price / wind windows"""
    p = SC.pool()
    rng = np.random.default_rng([T, OPERATIONS.index(name)])
    idx = rng.integers(0, len(p["dalmp_303"]) - T, N)[:, None] + np.arange(T)[None, :]
    da = p["dalmp_303"][idx]
    rt = da * rng.lognormal(0.0, 0.2, (N, T))
    cf = p["dacf_303"][idx]
    if name.startswith("wind_battery"):
        mode = name.split("wind_battery_")[1]
        disp = rng.uniform(0.0, 120.0, (N, T)) if mode == "tracker" else None
        rp = TP.wind_battery_operation_rparams(T, cf, 200.0, 25.0, 100.0, rng.uniform(0, 90000, N), rng.uniform(0, 5000, N), disp)
        cp = np.full((N, 1), 1e3) if mode == "tracker" else np.concatenate([da, rt, np.full((N, 1), 1e3)], axis=1)
        return certify(TP.wind_battery_operation(T, mode), cp, rp)
    if name.startswith("nuclear"):
        mode = name.split("nuclear_")[1]
        rp = np.concatenate([rng.uniform(0.0, 2e6, (N, 1)), rng.uniform(380.0, 520.0, (N, T))], axis=1)
        cp = np.full((N, 1), 4.0) if mode == "tracker" else np.concatenate([da, rt, np.full((N, 1), 4.0)], axis=1)
        return certify(TP.nuclear_operation(T, mode), cp, rp)
    rp = np.concatenate([cf * 200e3, np.full((N, 1), 200e3), rng.uniform(0.0, 150.0, (N, T))], axis=1)
    return certify(TP.wind_pem_operation(T), np.ones((N, 1)), rp)


@functools.lru_cache(maxsize=None)
def design(T=24, N=8):
    """battery sizing LPs (wind_battery_design): scarcity days make a battery worth building"""
    lmp, cf, W, _ = SC.c2(N, seed=8)
    lmp[::2] *= 40.0
    return certify(TP.wind_battery_design(T), lmp, TP.wind_battery_rparams(T, cf, W, 0.0))


SOLAR_SIZES = ("no_battery", "battery", "battery_pem")


def _solar_reference():
    from oracle import lp_models as L
    gold = json.load(open(Path(__file__).parent / "golden" / "solar_golden.json"))
    return np.array(gold["lmp_24"]), L.solar_default_series()


@functools.lru_cache(maxsize=None)
def solar(sizes, N=8, T=24):
    """PV + battery + hydrogen dispatch at fixed sizes (solar_battery_hydrogen, a band template), PV 200 MW: LP 0 is the reference's
    case, the others scale its prices (lognormal), loads (0.7 .. 1.2) and capacity factors (0.5 .. 1.0) per hour.  ``sizes``:
    no_battery (turbine and tank only), battery (50 MW / 200 MWh), battery_pem (and a 20 MW PEM).  The tank the reference sizes for
    its reserve (100 MW / (0.39 x 33.391) kg) backs 8.6e-14 kW less than 100 MW in exact arithmetic, so without a battery the
    night-time reserve rows make the reference's LP infeasible by that much: no_battery sizes the tank 1 % larger."""
    lmp0, d = _solar_reference()
    kw = {"no_battery": dict(tank_kg=1.01 * TP.solar_battery_hydrogen(T).meta["tank_kg"]),
          "battery": dict(batt_mw=50.0, batt_mwh=200.0),
          "battery_pem": dict(batt_mw=50.0, batt_mwh=200.0, pem_mw=20.0)}[sizes]
    rng = np.random.default_rng([T, 9, SOLAR_SIZES.index(sizes)])
    one = np.ones((1, T))
    lmp = np.tile(lmp0, T // 24) * np.vstack([one, rng.lognormal(0.0, 0.3, (N - 1, T))])
    load = np.tile(d["load_mw"], T // 24) * np.vstack([one, rng.uniform(0.7, 1.2, (N - 1, T))])
    cfs = np.tile(d["pv_cfs"], T // 24) * np.vstack([one, rng.uniform(0.5, 1.0, (N - 1, T))])
    return certify(TP.solar_battery_hydrogen(T, **kw), lmp, TP.solar_rparams(T, cfs, 200.0, load))


@functools.lru_cache(maxsize=None)
def solar_design(T=24, N=8, procs=1):
    """the PV + battery + hydrogen design LP over the baked template solar_battery_hydrogen_design(T, pv_cfs) with the reference's
    capacity factors (hour 12 of each day is sin(pi) = 1.2e-16, an entry of A that HiGHS drops): LP 0 is the reference's case, the
    others scale its prices (lognormal) and loads (0.7 .. 1.2) per hour"""
    lmp0, d = _solar_reference()
    rng = np.random.default_rng([T, 10])
    one = np.ones((1, T))
    lmp = np.tile(lmp0, T // 24) * np.vstack([one, rng.lognormal(0.0, 0.3, (N - 1, T))])
    load = 1e3 * np.tile(d["load_mw"], T // 24) * np.vstack([one, rng.uniform(0.7, 1.2, (N - 1, T))])
    return certify(TP.solar_battery_hydrogen_design(T, np.tile(d["pv_cfs"], T // 24)), lmp, load, procs)


SOLAR_PV = ("reference", "dyadic", "zero_hours", "all_zero", "cf_one", "reserve")


def solar_pv_series(T, N):
    """(lmp, load_mw, pv_cfs, reserve_mw) [N, T] of solar_design_pv, one row per SOLAR_PV case in that order, then perturbed series
    with zero hours: the reference's case; a series on the 1/64 grid (that LP is the baked template's LP bit for bit); a quarter of
    the hours exactly 0; an all-zero series; hours clipped at cf = 1; a perturbed reserve series"""
    from test_design_pv_series import dyadic_cfs
    lmp0, d = _solar_reference()
    rng = np.random.default_rng([T, 11])
    lmp = np.tile(lmp0, (N, T // 24))
    load = np.tile(d["load_mw"], (N, T // 24))
    cfs = np.tile(d["pv_cfs"], (N, T // 24))
    reserve = np.tile(d["reserve_mw"], (N, T // 24))
    lmp[2:] *= rng.lognormal(0.0, 0.3, (N - 2, T))
    load[2:] *= rng.uniform(0.7, 1.2, (N - 2, T))
    cfs[1] = dyadic_cfs(T, T)
    for k in [2] + list(range(len(SOLAR_PV), N)):
        cfs[k] *= rng.uniform(0.5, 1.0, T)
        cfs[k, rng.choice(T, T // 4, replace=False)] = 0.0
    cfs[3] = 0.0
    cfs[4] = np.minimum(1.0, 1.5 * cfs[4])
    reserve[5] *= rng.uniform(0.4, 1.0, T)
    return lmp, load, cfs, reserve


@functools.lru_cache(maxsize=None)
def solar_design_pv(T=24, N=8, procs=1):
    """the design LP with a PV and a reserve series per LP (solar_battery_hydrogen_design(T, None), per-problem matrix coefficients):
    the series of solar_pv_series"""
    lmp, load, cfs, reserve = solar_pv_series(T, N)
    return certify(TP.solar_battery_hydrogen_design(T, None), lmp, TP.solar_design_rparams(T, load, cfs, reserve), procs)


# ---------------------------------------------------------------------------------------------------------------------
# the check
# ---------------------------------------------------------------------------------------------------------------------
def errors(s: ExactSet, obj, x, y, cperm=None, rperm=None, kkt_rows=None):
    """the largest error of every measure of a kernel's (obj, x, y) on s (caller order: column j / row i is column cperm[j] /
    row rperm[i] of s.t):
      obj / lp      objective relative to max(1, |obj*|), and relative to sum |c_j x*_j| (the LP part; None when that is 0)
      x / y         element-wise, relative to each LP's |x*|_inf / |y*|_inf, on the LPs unique in x with r_margin >= R_MARGIN / unique
                    in y with x_margin >= X_MARGIN (None if there are none): the planted suite's margins.  An LP unique in x whose
                    smallest nonbasic reduced cost is 1e-6 |c|_inf has x_j ~ mu / r_j off its bound (2.5e-5 seen in C2 on an H100)
      fixed         |x_j - x*_j| on fixed columns with |r*_j| >= R_MARGIN |c|_inf, relative to max(1, |x*|_inf)
      inside        |r_j(y)| on inside columns at least X_MARGIN max(1, |x*|_inf) from both bounds, relative to |c|_inf
      primal, bound, dual_inf, gap   kkt_residuals of the LPs ``kkt_rows`` (default all; dual_inf and gap over LPs whose LP part
                    is not identically 0)"""
    ci = np.arange(s.t.n) if cperm is None else np.argsort(cperm)      # template column j is caller column ci[j]
    ri = np.arange(s.t.m) if rperm is None else np.argsort(rperm)
    xt, yt = x[:, ci], y[:, ri]
    eo = np.abs(obj - s.obj) / np.maximum(1.0, np.abs(s.obj))
    nz = s.lp_mag > 0
    el = np.abs(obj - s.obj)[nz] / s.lp_mag[nz]
    ux, uy = s.unique_x & (s.r_margin >= R_MARGIN), s.unique_y & (s.x_margin >= X_MARGIN)
    out = dict(obj=float(eo.max()), lp=float(el.max()) if nz.any() else None,
               x=rel(xt[ux], s.x[ux]) if ux.any() else None, y=rel(yt[uy], s.y[uy]) if uy.any() else None)
    xs = np.maximum(1.0, np.abs(s.x).max(1))
    A = s.t.A.tocsc() if s.t.amap is None else None
    ef = ei = 0.0
    for k in range(len(s)):
        big = s.fixed[k] & (np.abs(s.r[k]) >= R_MARGIN * s.csc[k])
        if big.any():
            ef = max(ef, float(np.abs(xt[k, big] - s.x[k, big]).max() / xs[k]))
        if not nz[k] or s.csc[k] == 0.0:
            continue
        u = s.u[k]
        d = np.minimum(s.x[k], np.where(np.isfinite(u), u - s.x[k], np.inf))
        deep = s.inside[k] & (d >= X_MARGIN * xs[k])
        if deep.any():
            Ak = A if A is not None else s.t.matrix(s.rparams[k]).tocsc()
            c = s.t.instantiate(s.cparams[k], s.rparams[k])[0]
            rk = c - Ak.T @ yt[k]
            ei = max(ei, float(np.abs(rk[deep]).max() / s.csc[k]))
    out.update(fixed=ef, inside=ei)
    rows = range(len(s)) if kkt_rows is None else kkt_rows
    kk = [kkt_residuals(s.t, s.cparams[i], s.rparams[i], xt[i], yt[i], lp_zero=not nz[i]) for i in rows]
    for key in ("primal", "bound", "dual_inf", "gap"):
        v = [d[key] for d in kk if d[key] is not None]
        out[key] = max(v) if v else None
    return out


def check_exact(s: ExactSet, obj, status, x, y, cperm=None, rperm=None, kkt_rows=None, what="", obj_rel=OBJ_REL):
    """asserts status OPTIMAL and every measure of ``errors`` within the planted suite's bars (planted_stage: OBJ_REL, XY_REL,
    KKT_*); the fixed / inside measures use XY_REL.  ``obj_rel`` replaces the objective bar for a set whose larger objective error is
    recorded where it is checked.  Returns the errors."""
    assert (status == 0).all(), (what, np.unique(status, return_counts=True))
    e = errors(s, obj, x, y, cperm, rperm, kkt_rows)
    le = lambda v, bar: v is None or v <= bar
    assert le(e["obj"], obj_rel) and le(e["lp"], obj_rel), (what, e)
    assert le(e["x"], XY_REL) and le(e["y"], XY_REL) and e["fixed"] <= XY_REL and e["inside"] <= XY_REL, (what, e)
    assert max(e["primal"], e["bound"]) <= KKT_PRIMAL and le(e["dual_inf"], KKT_DUAL) and le(e["gap"], KKT_GAP), (what, e)
    return e


def fmt(e):
    return {k: ("n/a" if v is None else f"{v:.1e}") for k, v in e.items()}
