"""LPs with a known, nondegenerate optimum for the stage kernels (test infrastructure, no GPU).

``planted_wb``: price / wind data for the real ``templates.wind_battery(T)`` template, so that the wind + battery stage kernels
(stage 2, stage v1, the long-horizon kernel) run on their own hard-wired structure.  Every LP is one charge / discharge cycle whose
optimum is unique in x and y; each is certified by ``exact_lp.exact_optimum`` and only certified LPs are kept.

``planted_chain``: storage-chain LPs for the descriptor-driven chain kernel (csrc/dsp_stage_chain1.cuh) with the dyadic
construction of planted_lp.py, so that b, c and the objective are exact in binary64 and x*, y* are known by construction.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import scipy.sparse as sp

from dispatches_b200 import templates as TP
from dispatches_b200.lp_template import INF, LPTemplate, detect_chain1
from exact_lp import NotCertified, exact_optimum, kkt_residuals
from planted_lp import _dy, rel


# Bounds on a kernel's answer against the exact optimum, shared by the emulator (CPU) and GPU tests.  The kernels stop at
# res < feas_tol and gap < tol (1e-9 each), or at res < 10 feas_tol and gap < 10 tol once complementarity has converged, where
# res is the larger of the primal and dual residual relative to 1 + the scaled |b| / |c|, and gap the relative gap of the scaled
# LP.  A third, relaxed branch accepts res < 100 feas_tol and gap < 1000 tol; these bounds are set so that an LP it lets through
# with more than the second branch's error fails.
OBJ_REL = 1e-7       # objective (and its LP part c'x) vs the exact optimum: 10x the second branch's gap, as for the band kernel
XY_REL = 1e-6        # x and y element-wise, relative to each LP's |.|_inf, as for the band kernel.  An interior-point iterate
                     # stops with x_j ~ mu / r_j on a nonbasic column, so the error grows as the reduced-cost margin shrinks: the
                     # base cycle keeps r_margin >= 1e-3 and x_margin >= 1e-2 (test_planted_stage.py asserts both).  Largest
                     # errors seen: x 4e-7 on the emulator, 9.6e-7 on an H100 (long kernel, T = 200, r_margin 4.2e-3) -- the
                     # tightest case of the suite; y at most 1.5e-7
KKT_PRIMAL = 1e-8    # |A x - b| and bound violation: the second branch's 10 feas_tol (the relaxed branch allows 1e-7)
KKT_DUAL = 1e-8      # max(-r_j, 0) over unbounded columns: the dual residual of the second branch (10 feas_tol)
KKT_GAP = 1e-7       # duality gap relative to sum |c_j x_j| (>= |c'x|): 10x the second branch's 10 tol (the relaxed one allows 1e-6)


@dataclasses.dataclass
class PlantedStage:
    t: LPTemplate
    cparams: np.ndarray        # [N, Pc]
    rparams: np.ndarray        # [N, Pr]
    x: np.ndarray              # [N, n] exact optimum, template column order
    y: np.ndarray              # [N, m] exact row duals, template row order
    obj: np.ndarray            # [N] c'x* + k
    lp_mag: np.ndarray         # [N] sum_j |c_j x*_j|
    drawn: int = 0             # LPs drawn to get the N kept
    x_margin: float = math.inf
    r_margin: float = math.inf

    def tile(self, N, seed=0):
        """N LPs: the batch repeated in a random permutation (every copy bitwise equal to its first copy)"""
        k = np.random.default_rng(seed).permutation(np.resize(np.arange(len(self.obj)), N))
        return dataclasses.replace(self, cparams=self.cparams[k], rparams=self.rparams[k], x=self.x[k], y=self.y[k],
                                   obj=self.obj[k], lp_mag=self.lp_mag[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# wind + battery
# ---------------------------------------------------------------------------------------------------------------------
def _wb_draw(T, rng, soc):
    """prices and wind of one charge / discharge cycle.

    Base cycle (soc=False): n <= 3 full-power charge hours (hour 0 among them, so the battery is never empty and idle) and n
    discharge hours at the end of the horizon, at prices in [100, 200].  With round-trip losses the cycle fills n P / 0.95 ...
    empties in floor(0.9025 n) full hours and one partial one, the cheapest discharge hour: that partial discharge is the one
    basic battery flow.  Every other hour sits in the battery's no-trade band (0.91 - 0.99 x the cheapest discharge price, above
    the 0.9025 x at which charging would pay), charge hours at 0.3 - 0.85 x.  Wind x cf is 1.2 - 4 x P in every hour, so the
    grid sale is basic everywhere.

    soc=True: five cheap charge hours (0 - 4) fill the battery to capacity at hour 4 (5 x 0.95 P > 4 P), so the soc_bound row of
    hour 4 binds and its dual is nonzero; discharge starts at hour 5 (so the bound binds in that hour only) and ends in the last
    three hours.  The most expensive charge hour charges partially."""
    P = float(rng.integers(40, 800)) * 1000.0
    lmp = np.empty(T)
    if soc:
        charge = list(range(5))
        dis = [5] + list(range(T - 3, T))
    else:
        n = int(rng.integers(1, min(3, T // 2) + 1))
        charge = [0] + sorted(rng.choice(np.arange(1, T - n), n - 1, replace=False).tolist()) if n > 1 else [0]
        dis = list(range(T - n, T))
    lmp[dis] = rng.uniform(100.0, 200.0, len(dis))
    pmin = lmp[dis].min()
    idle = [h for h in range(T) if h not in charge and h not in dis]
    lmp[idle] = pmin * rng.uniform(0.91, 0.99, len(idle))
    lmp[charge] = pmin * rng.uniform(0.3, 0.85, len(charge))
    wcf = P * rng.uniform(1.2, 4.0, T)
    W = float(rng.integers(2000, 4000)) * 1000.0
    return lmp, np.r_[wcf, P, W]


def planted_wb(T, N, seed=0, soc=False, min_rate=0.9):
    """N certified wind + battery LPs over templates.wind_battery(T) (cparams = prices, rparams = [wind x cf (T), P, W]).  Draws
    until N LPs are certified unique in x and y and asserts that at least ``min_rate`` of the draws were."""
    t = TP.wind_battery(T)
    rng = np.random.default_rng([T, seed, int(soc)])
    cps, rps, xs, ys, objs, mags = [], [], [], [], [], []
    drawn = 0
    xm = rm = math.inf
    while len(objs) < N:
        drawn += 1
        lmp, rp = _wb_draw(T, rng, soc)
        try:
            e = exact_optimum(t, lmp, rp)
        except NotCertified:
            continue
        if not (e.unique_x and e.unique_y):
            continue
        cps.append(lmp); rps.append(rp); xs.append(e.x); ys.append(e.y); objs.append(e.obj); mags.append(e.lp_mag)
        xm, rm = min(xm, e.x_margin), min(rm, e.r_margin)
        if drawn >= 4 * N + 20:
            break
    assert len(objs) >= min_rate * drawn, f"planted_wb(T={T}, soc={soc}): {len(objs)} of {drawn} draws certified"
    return PlantedStage(t, np.array(cps), np.array(rps), np.array(xs), np.array(ys), np.array(objs), np.array(mags), drawn, xm, rm)


# ---------------------------------------------------------------------------------------------------------------------
# storage chain
# ---------------------------------------------------------------------------------------------------------------------
def planted_chain(T, NF, seed=0, N=1, bounded="mixed", c_scale=1.0, b_scale=1.0):
    """N planted single-storage-chain LPs over one template.

    One equality row per period; NF (2 or 3) flow columns per row, some rows with fewer; one state column per period t < T - 1
    in rows t and t + 1 with independent coefficients; the last row has no state.  The basis is a forest: the rows are cut into
    segments, each segment has one basic flow and its internal states basic, the states between segments and every other flow
    are nonbasic at 0 or u.  Each segment is a tree, so B is nonsingular.  x* first, then b = A x*, then y* and r (r_B = 0,
    |r_N| >= 1/8 with the sign complementarity asks for), then c = A'y* + r: every number is dyadic, so the data and the
    objective are exact in binary64.  cparams = c (n), rparams = [b (m) | u of the bounded columns].  ``c_scale`` / ``b_scale``
    scale c and y* / b, u and x*."""
    rng = np.random.default_rng([T, NF, seed, {"mixed": 0, "all": 1, "none": 2}[bounded]])
    # ---- columns in caller order: (rows, values, kind)
    cols = []
    full_row = int(rng.integers(0, T - 1))                   # a row before the last with all NF flows: detect_chain1 sees NF
    for t in range(T):
        nf = NF if t == full_row else int(rng.integers(1, NF + 1))
        for _ in range(nf):
            cols.append(([t], [float(_dy(rng, 0.5, 2, 2)) * rng.choice([-1.0, 1.0])], "flow", t))
        if t < T - 1:
            cols.append(([t, t + 1], [float(_dy(rng, 0.5, 2, 2)) * rng.choice([-1.0, 1.0]),
                                      float(_dy(rng, 0.5, 2, 2)) * rng.choice([-1.0, 1.0])], "state", t))
    order = rng.permutation(len(cols))
    cols = [cols[k] for k in order]
    n, m = len(cols), T
    # ---- basis: segments of 1 - 4 rows, one basic flow each, internal states basic
    basic = np.zeros(n, bool)
    cuts, s = [], 0
    while s < T:
        e = min(T, s + int(rng.integers(1, 5)))
        cuts.append((s, e)); s = e
    for s, e in cuts:
        fl = [j for j, c in enumerate(cols) if c[2] == "flow" and s <= c[3] < e]
        basic[fl[int(rng.integers(0, len(fl)))]] = True
        for j, c in enumerate(cols):
            if c[2] == "state" and s <= c[3] < e - 1:
                basic[j] = True
    assert basic.sum() == m
    ri, ci, vv = [], [], []
    for j, (rows, vals, _, _) in enumerate(cols):
        ri += rows; ci += [j] * len(rows); vv += vals
    A = sp.csr_matrix((vv, (ri, ci)), shape=(m, n))
    A.sort_indices()
    fin = np.ones(n, bool) if bounded == "all" else np.zeros(n, bool) if bounded == "none" else rng.random(n) < 0.5
    fidx = np.flatnonzero(fin)
    nb = len(fidx)
    Pc, Pr = n, m + nb
    Cmap = sp.identity(n, format="csr")
    Bmap = sp.csr_matrix((np.ones(m), (np.arange(m), np.arange(m))), shape=(m, Pr))
    Umap = sp.csr_matrix((np.ones(nb), (fidx, m + np.arange(nb))), shape=(n, Pr))
    u0 = np.full(n, INF); u0[fidx] = 0.0
    o0 = float(_dy(rng, -8, 8, 3)); omap = np.r_[_dy(rng, -1, 1, 3, m), np.zeros(nb)]; ocmap = _dy(rng, -1, 1, 3, Pc)
    CP = np.zeros((N, Pc)); RP = np.zeros((N, Pr)); X = np.zeros((N, n)); Y = np.zeros((N, m)); OBJ = np.zeros(N); MAG = np.zeros(N)
    for k in range(N):
        u = np.full(n, INF); u[fin] = _dy(rng, 2, 8, 2, nb) * b_scale
        x = np.zeros(n)
        at_u = fin & ~basic & (rng.random(n) < 0.5)
        x[at_u] = u[at_u]
        x[basic & ~fin] = _dy(rng, 1, 4, 6, int((basic & ~fin).sum())) * b_scale
        x[basic & fin] = u[basic & fin] * _dy(rng, 0.125, 0.875, 6, int((basic & fin).sum()))
        b = A @ x
        y = _dy(rng, -2, 2, 4, m) * c_scale
        r = _dy(rng, 0.125, 10, 3, n) * c_scale
        r[at_u] = -r[at_u]; r[basic] = 0.0
        c = A.T @ y + r
        CP[k] = c; RP[k, :m] = b; RP[k, m:] = u[fidx]
        X[k], Y[k] = x, y
        OBJ[k] = math.fsum(list(c * x) + [o0] + list(omap * RP[k]) + list(ocmap * c))
        MAG[k] = math.fsum(np.abs(c * x))
    t = LPTemplate(f"planted_chain(T={T},NF={NF})", A, np.zeros(m), Bmap, np.zeros(n), Cmap, u0, Umap, o0, omap, ocmap,
                   np.zeros(n), np.ones(n), [f"x{j}" for j in range(n)], [f"r{i}" for i in range(m)])
    t.finalize()
    d = detect_chain1(t)
    assert d is not None and d["NF"] == NF and d["T"] == T, d
    cpos = np.array([int(nm[1:]) for nm in t.col_names]); rpos = np.array([int(nm[1:]) for nm in t.row_names])
    # the maps follow the template's column order; cparams / rparams stay in the generator's (the maps index them)
    return PlantedStage(t, CP, RP, X[:, cpos], Y[:, rpos], OBJ, MAG, N)


# chain test cases: lanes per LP (chain1_lanes in csrc/dsp_lp.cu) -> a horizon that leaves lanes / periods idle, or fills them
CHAIN_T = {4: 11, 8: 24, 16: 37, 32: 96}
# scaled chain data (c, b x 2^+-20), as planted_lp.VARIANTS for the band kernel
CHAIN_VARIANTS = {"c_up": dict(c_scale=2.0 ** 20), "c_down": dict(c_scale=2.0 ** -20), "b_up": dict(b_scale=2.0 ** 20),
                  "b_down": dict(b_scale=2.0 ** -20)}


def chain_lanes(T):
    """lanes per LP of the chain kernel (chain1_lanes in csrc/dsp_lp.cu)"""
    return 4 if T <= 12 else 8 if T <= 24 else 16 if T <= 48 else 32


def chain_smem_bytes(NF, P=3):
    """shared memory per warp of the chain kernel (chain1::Smem<NF, P>::doubles_per_warp x 8 in csrc/dsp_stage_chain1.cuh)"""
    na_full, na_int = 7 * (NF + 1) + 3, 3
    return (na_full * P + na_int * (P - 1)) * 32 * 8


def check(p: PlantedStage, obj, status, x, y, t=None, cperm=None, rperm=None, kkt_rows=None, what=""):
    """status OPTIMAL, objective (whole and LP part) within OBJ_REL of the exact optimum, x / y within XY_REL in the caller order
    (template ``t``, default p.t, whose column j / row i is column cperm[j] / row rperm[i] of p.t), and the KKT residuals of the
    LPs ``kkt_rows`` (default: all) within KKT_*; returns the largest (objective, x, y) errors and KKT residuals"""
    assert (status == 0).all(), (what, np.unique(status, return_counts=True))
    eo = np.abs(obj - p.obj) / np.maximum(1.0, np.abs(p.obj))
    el = np.abs(obj - p.obj) / np.maximum(p.lp_mag, 1e-300)
    assert eo.max() <= OBJ_REL and el.max() <= OBJ_REL, (what, eo.max(), el.max())
    xr = p.x if cperm is None else p.x[:, cperm]
    yr = p.y if rperm is None else p.y[:, rperm]
    ex, ey = rel(x, xr), rel(y, yr)
    assert ex <= XY_REL and ey <= XY_REL, (what, ex, ey)
    t = p.t if t is None else t
    k = [kkt_residuals(t, p.cparams[i], p.rparams[i], x[i], y[i]) for i in (range(len(obj)) if kkt_rows is None else kkt_rows)]
    kk = {key: max(d[key] for d in k) for key in ("primal", "bound", "dual_inf", "gap")}
    assert max(kk["primal"], kk["bound"]) <= KKT_PRIMAL and kk["dual_inf"] <= KKT_DUAL and kk["gap"] <= KKT_GAP, (what, kk)
    return dict(obj=float(max(eo.max(), el.max())), x=ex, y=ey, **kk)
