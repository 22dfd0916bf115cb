"""Pyomo solver plugin ``SolverFactory("b200ipm")`` -- SURVEY.md §8(f)-1, import-guarded.

Replaces ``pyo.SolverFactory("cbc")`` at the reference's call sites (wind_battery_LMP.py:266-267,
wind_battery_PEM_LMP.py:296-298, price_taker_analysis.py:365,403) without touching the model builders: the built
Pyomo model is walked ONCE (``extract``: pyomo -> plain rows / bounds / cost arrays; ``lp_template.standard_form``: pure,
tested without pyomo on the oracle's reference-shaped raw LPs, tests/test_standard_form.py) into an LPTemplate, handed to the
library as a plain standard-form LP (dsp_lp_template_create_csr), then solved on the GPU -- for the model as it stands (batch of 1, values
written back into the Vars like any Pyomo solver) or for a whole batch of values of its mutable Params
(``batch_params={param: array[N]}``, e.g. every block's ``lmp_signal``, wind_battery_LMP.py:234,243-244).

pyomo is NOT installed in the build image (SURVEY.md §0.4), so this module is exercised only where pyomo exists;
``import dispatches_b200.pyomo_plugin`` never fails, ``available()`` reports the truth.
"""
from __future__ import annotations

import numpy as np

from .lp_template import INF, model_duals, model_reduced_costs, model_values, standard_form
from .solver import INFEASIBLE, MAX_ITER, OPTIMAL, BatchLPSolver, LPResult

try:                                            # pragma: no cover - pyomo absent in the build image
    import pyomo.environ as pyo
    from pyomo.opt import SolverFactory, SolverResults, SolverStatus, TerminationCondition
    from pyomo.repn import generate_standard_repn
    HAVE_PYOMO = True
except Exception:                               # noqa: BLE001
    HAVE_PYOMO = False


def extract(model, batch_params=None):
    """The pyomo half of the walker: the active linear Constraints / Objective of ``model`` as plain arrays for
    lp_template.standard_form().  Every active Constraint / the active Objective is reduced with generate_standard_repn (fixed
    Vars fold into the constant).  Mutable Params listed in ``batch_params`` are handled by one finite difference each (the
    dependence is affine by construction): cost coefficients, right-hand sides and Var bounds may depend on them, constraint
    matrix coefficients may not (the matrix is shared by the batch)."""
    if not HAVE_PYOMO:
        raise RuntimeError("pyomo is not installed: the b200ipm plugin needs it to walk the model")
    batch_params = list(batch_params or [])
    vars_, vid = [], {}

    def col(v):
        k = id(v)
        if k not in vid:
            vid[k] = len(vars_)
            vars_.append(v)
        return vid[k]

    cons = list(model.component_data_objects(pyo.Constraint, active=True, descend_into=True))
    objs = list(model.component_data_objects(pyo.Objective, active=True, descend_into=True))
    if len(objs) != 1:
        raise ValueError("exactly one active Objective expected")

    def snapshot():
        rows, lo, hi = [], [], []
        for c in cons:
            r = generate_standard_repn(c.body, compute_values=True)
            if not r.is_linear():
                raise ValueError(f"constraint {c.name} is not linear: b200ipm solves LPs only")
            rows.append({col(v): float(a) for v, a in zip(r.linear_vars, r.linear_coefs)})
            lo.append(-INF if c.lower is None else float(pyo.value(c.lower)) - float(r.constant))
            hi.append(INF if c.upper is None else float(pyo.value(c.upper)) - float(r.constant))
        r = generate_standard_repn(objs[0].expr, compute_values=True)
        if not r.is_linear():
            raise ValueError("objective is not linear")
        cost = {col(v): float(a) for v, a in zip(r.linear_vars, r.linear_coefs)}
        return rows, np.array(lo), np.array(hi), cost, float(r.constant)

    def bounds():
        lb = np.array([(-INF if v.lb is None else float(v.lb)) for v in vars_])
        ub = np.array([(INF if v.ub is None else float(v.ub)) for v in vars_])
        return lb, ub

    rows, lo, hi, cost, c0 = snapshot()
    n0 = len(vars_)
    lb, ub = bounds()
    P = len(batch_params)
    dcost = np.zeros((n0, P)); dlo = np.zeros((len(rows), P)); dhi = np.zeros_like(dlo); dc0 = np.zeros(P)
    dlb = np.zeros((n0, P)); dub = np.zeros((n0, P))
    for k, p in enumerate(batch_params):
        old = pyo.value(p)
        p.set_value(old + 1.0)
        try:
            rows1, lo1, hi1, cost1, c01 = snapshot()
            lb1, ub1 = bounds()
        finally:
            p.set_value(old)
        if len(vars_) != n0 or any(r1 != r0 for r1, r0 in zip(rows1, rows)):
            raise ValueError(f"Param {p.name} enters the constraint matrix: it cannot be batched")
        for j in range(n0):
            dcost[j, k] = cost1.get(j, 0.0) - cost.get(j, 0.0)
        fin = np.isfinite(lo); dlo[fin, k] = lo1[fin] - lo[fin]
        fin = np.isfinite(hi); dhi[fin, k] = hi1[fin] - hi[fin]
        fin = np.isfinite(lb); dlb[fin, k] = lb1[fin] - lb[fin]
        fin = np.isfinite(ub); dub[fin, k] = ub1[fin] - ub[fin]
        dc0[k] = c01 - c0
    p0 = np.array([pyo.value(p) for p in batch_params], float)
    sense = 1.0 if objs[0].sense == pyo.minimize else -1.0
    return dict(rows=rows, lo=lo, hi=hi, lb=lb, ub=ub, cost=cost, c0=c0, sense=sense, var_names=[v.name for v in vars_],
                p0=p0, dcost=dcost, dlo=dlo, dhi=dhi, dlb=dlb, dub=dub, dc0=dc0), vars_, cons


def walk_model(model, batch_params=None):
    """Pyomo model -> (LPTemplate, Vars, Constraints, p0): extract() + the pure lp_template.standard_form() (free Vars are split,
    ranged rows get a bounded slack, maximisation flips the cost, arcs / link equalities are presolved away)."""
    data, vars_, cons = extract(model, batch_params)
    t = standard_form(name="pyomo:" + str(getattr(model, "name", "model")), **data)
    return t, vars_, cons, data["p0"]


class B200IPM:
    """Object with the part of Pyomo's solver interface the reference uses (SURVEY.md 8b): ``available()``, ``options``,
    ``solve(model, tee=...)`` writing Var values (and ``model.dual`` / ``model.rc`` when the model declares an IMPORT Suffix of that
    name) back, returning SolverResults with solver.status / termination_condition.  ``options={"sensitivities": True}`` adds
    ``res.batch["d_params"]`` [N, P]: d objective / d every batched Param (a subgradient where the optimum is not unique), from the
    GPU post-pass dsp_lp_sensitivities.  ``options={"crossover": True}`` (templates of up to 1024 rows) returns a vertex of every LP, as a
simplex solver such as CBC does: a plain solve writes the vertex into the Vars, ``model.dual`` and ``model.rc`` (presolve's
substitutions, splits and flips are affine bijections, so a vertex of the template is a vertex of the model); a batched solve returns
the vertex in ``res.batch`` (``obj``, ``x``, ``duals``) with the basis and crossover status in ``res.batch["crossover"]``.  An LP
whose crossover does not end OPTIMAL keeps its interior-point solution, and ``res.solver.message`` says so.
``options={"ranging": True}`` implies crossover and adds ``res.batch["param_ranges"]`` [N, P, 2]: for every batched Param, all others
fixed, the absolute [lo, hi] values over which the LP's vertex stays optimal (GPU post-pass dsp_lp_ranging along the Param's axis; NaN
for an LP whose crossover did not end OPTIMAL and for a Param that is a coefficient of the constraint matrix)."""

    def __init__(self, **kw):
        self.options = dict(tol=1e-9, feas_tol=1e-9, max_iter=60)
        self.options.update(kw)

    def available(self, exception_flag=True):
        try:
            from .solver import load_library
            import torch
            load_library()
            ok = HAVE_PYOMO and torch.cuda.is_available()
        except Exception:                       # noqa: BLE001
            ok = False
        if not ok and exception_flag:
            raise RuntimeError("b200ipm needs pyomo, libdsp_lp.so and a CUDA device (there is no CPU fallback)")
        return ok

    def solve(self, model, tee=False, batch_params=None, options=None, **_):
        opts = dict(self.options); opts.update(options or {})
        t, vars_, cons, p0 = walk_model(model, batch_params=list((batch_params or {}).keys()))
        # options["kernel"]: a solver.KERNEL_* choice, e.g. KERNEL_BAND_SPLIT for a long horizon (unset: the library's default)
        kern = {"kernel": int(opts["kernel"])} if opts.get("kernel") is not None else {}
        sol = BatchLPSolver(t, tol=opts["tol"], feas_tol=opts["feas_tol"], max_iter=opts["max_iter"], native_setup=True, **kern)
        if batch_params:
            pv = np.column_stack([np.asarray(batch_params[p], float) for p in batch_params])
        else:
            pv = p0[None, :] if p0.size else np.zeros((1, 0))
        sense = t.meta["sense"]
        d_params = vertex = param_ranges = None
        message = None
        if opts.get("sensitivities") or opts.get("crossover") or opts.get("ranging"):
            # the device path: the same Param vector is cparams and rparams, so d obj / d Param = d_cparams + d_rparams
            import torch
            dev = torch.device("cuda", torch.cuda.current_device())
            pvt = torch.as_tensor(np.ascontiguousarray(pv, float), device=dev)
            rd = sol.solve(pvt, pvt if t.Pr else None, want_x=True, want_y=True)
            if opts.get("crossover") or opts.get("ranging"):
                v = sol.crossover(pvt, pvt if t.Pr else None, rd)
                ok = v.status == OPTIMAL
                rd = LPResult(torch.where(ok, v.obj, rd.obj), rd.status, rd.iters, torch.where(ok[:, None], v.x, rd.x),
                              torch.where(ok[:, None], v.y, rd.y))
                vertex = {k: getattr(v, k).cpu().numpy() for k in ("status", "pivots", "col_status", "row_basic")}
                lost = np.flatnonzero((vertex["status"] != OPTIMAL) & (rd.status.cpu().numpy() == OPTIMAL))
                if lost.size:
                    message = (f"crossover did not reach a vertex for {lost.size} LP(s) (first: {int(lost[0])}, crossover status "
                               f"{int(vertex['status'][lost[0]])}): their interior-point solution is loaded")
            if opts.get("ranging"):
                # Param k moves its cparams and its rparams entry together: the direction (e_k, e_k)
                P = pv.shape[1]
                lo = hi = np.zeros((pv.shape[0], 0))
                if P:
                    eye = torch.eye(P, dtype=torch.float64, device=dev)
                    g = sol.ranging(pvt, pvt if t.Pr else None, v, eye, eye if t.Pr else None)
                    lo, hi = g.theta_lo.cpu().numpy(), g.theta_hi.cpu().numpy()
                param_ranges = np.stack([pv + lo, pv + hi], axis=-1)
            if opts.get("sensitivities"):
                g = sol.sensitivities(pvt, pvt if t.Pr else None, rd, want_rc=False)
                d_params = sense * (g.d_cparams + g.d_rparams).cpu().numpy()
            r = LPResult(*(a.cpu().numpy() for a in (rd.obj, rd.status, rd.iters, rd.x, rd.y)))
        else:
            r = sol.solve_host(pv, pv if t.Pr else None, want_x=True, want_y=True)
        xm = model_values(t, r.x, pv)
        ym = model_duals(t, r.y)
        if pv.shape[0] == 1:                    # plain solver behaviour: write back into the Vars (and the dual Suffix)
            for j, v in enumerate(vars_):
                v.set_value(float(xm[0, j]), skip_validation=True)
                v.stale = False
            dual = getattr(model, "dual", None)
            if dual is not None and hasattr(dual, "import_enabled") and dual.import_enabled():
                for i, c in enumerate(cons):
                    dual[c] = float(ym[0, i])
            rc = getattr(model, "rc", None)
            if rc is not None and hasattr(rc, "import_enabled") and rc.import_enabled():
                rcm = model_reduced_costs(t, r.y, pv)
                for j, v in enumerate(vars_):
                    rc[v] = float(rcm[0, j])
        res = SolverResults()
        worst = int(r.status.max())
        res.solver.status = {OPTIMAL: SolverStatus.ok, MAX_ITER: SolverStatus.warning}.get(worst, SolverStatus.error)
        res.solver.termination_condition = {OPTIMAL: TerminationCondition.optimal, MAX_ITER: TerminationCondition.maxIterations,
                                            INFEASIBLE: TerminationCondition.infeasible}.get(worst, TerminationCondition.error)
        res.problem.lower_bound = res.problem.upper_bound = float(sense * r.obj[0])
        res.batch = dict(obj=sense * r.obj, status=r.status, iters=r.iters, x=xm, duals=ym, var_names=[v.name for v in vars_])
        if d_params is not None:
            res.batch["d_params"] = d_params
        if vertex is not None:
            res.batch["crossover"] = vertex
        if param_ranges is not None:
            res.batch["param_ranges"] = param_ranges
        if message is not None:
            res.solver.message = message
        if tee:
            print(f"b200ipm: {pv.shape[0]} LP(s), m={t.m} n={t.n} w={t.w}, iterations max {int(r.iters.max())}")
        return res


if HAVE_PYOMO:                                  # pragma: no cover
    try:
        SolverFactory.register("b200ipm", doc="H100 batched interior-point LP solver")(B200IPM)
    except Exception:                           # noqa: BLE001
        pass
