"""LPs and starting points that drive every path of the crossover's simplex (dsp_lp_crossover, csrc/dsp_crossover.cuh), for the
emulator and GPU tests of tests/test_crossover_paths*.py (test infrastructure, no GPU).

The crossover's own suites start from a near-optimal interior point of a dispatch LP, where the cleanup has next to nothing to do.
These inputs give it work:
  - assignment(k): the k x k assignment LP (rows: every worker and every job assigned once, 0 <= x <= 1), integer costs as cparams.
    Its 2k rows have rank 2k - 1, so one artificial always stays basic (a redundant row).  From x = 0 the all-artificial basis is
    dual feasible and primal infeasible: dual simplex pivots, long runs of degenerate ones (Bland's rule) and reinversions.  From the
    identity permutation (feasible, maximally degenerate) the basis is primal feasible and dual infeasible: degenerate primal pivots
    and bound flips.  Its optimum is linear_sum_assignment's, and with integer costs the objective is an exact integer.
  - planted LPs (tests/planted_lp.py), whose unique optimum x* is known: started from x* with the nonbasic columns at 0 moved to
    their upper bounds (bound flips back to x*), and from x* with a third of its basic columns set to 0 (primal and dual infeasible
    after the push: DSP_NUMERICAL, as include/dsp_lp.h documents).
  - planted LPs sized to either side of the crossover's placement boundary (its work region in shared memory, or in the workspace)
    and to m = 1024, the largest m the crossover takes.
"""
from __future__ import annotations

import dataclasses

import numpy as np

import exact_lp as E
from dispatches_b200.lp_template import TemplateBuilder
import planted_lp as PL

FIELDS = ("obj", "x", "y", "col_status", "row_basic", "status", "pivots")     # the crossover's outputs
MAX_M = 1024                # dsp_lp_crossover / dsp_lp_ranging take m <= 1024
XO_THREADS = 256            # xo::kMaxThreads: the entries of xo::Shared's reduction arrays


@dataclasses.dataclass
class Inputs:
    """one batch for the crossover: a template, its parameters and the interior-point-like (status, x, y) it starts from"""
    t: object
    cparams: np.ndarray
    rparams: np.ndarray | None
    status: np.ndarray
    x: np.ndarray
    y: np.ndarray


_assign = {}


def assignment_template(k):
    """the k x k assignment LP: column x{i}_{j} (worker i does job j, 0 <= x <= 1, cost cparams[i k + j]), rows w{i} and j{j}"""
    if k not in _assign:
        B = TemplateBuilder(f"assignment({k})", k * k, 0)
        xs = [[B.var(f"x{i}_{j}", ub=1.0) for j in range(k)] for i in range(k)]
        for i in range(k):
            for j in range(k):
                B.cost(xs[i][j], (0.0, {i * k + j: 1.0}))
        for i in range(k):
            B.eq(f"w{i}", {xs[i][j]: 1.0 for j in range(k)}, 1.0)
        for j in range(k):
            B.eq(f"j{j}", {xs[i][j]: 1.0 for i in range(k)}, 1.0)
        _assign[k] = B.build()
    return _assign[k]


def assignment_costs(k, N, hi, seed=0):
    """[N, k, k] integer costs in 0 .. hi"""
    return np.random.default_rng(seed).integers(0, hi + 1, size=(N, k, k)).astype(float)


def assignment(k, N, hi, start, seed=0):
    """N k x k assignment LPs with costs in 0 .. hi, started from x = 0 (start="zero") or the identity permutation
    (start="identity").  The cparams are the costs in template column order."""
    t = assignment_template(k)
    cost = assignment_costs(k, N, hi, seed)
    cp = np.zeros((N, t.Pc))
    cp[:, :] = cost.reshape(N, k * k)                     # cparams[i k + j] is the cost of x{i}_{j}, whatever the column order
    x = np.zeros((N, t.n))
    if start == "identity":
        x[:, [t.column(f"x{i}_{i}") for i in range(k)]] = 1.0
    elif start != "zero":
        raise ValueError(start)
    return Inputs(t, cp, None, np.zeros(N, np.int32), x, np.zeros((N, t.m)))


def assignment_optimum(cost):
    """the assignment objective of every [k, k] cost matrix (scipy.optimize.linear_sum_assignment), exact for integer costs"""
    from scipy.optimize import linear_sum_assignment
    out = []
    for c in cost:
        r, q = linear_sum_assignment(c)
        out.append(float(c[r, q].sum()))
    return np.array(out)


def planted_basis(p, k=0):
    """(col_status [n] int8, row_basic [m] bool) of the planted optimum of LP k: its owned columns basic, the others at their bound"""
    c, b, u, _ = p.t.instantiate(p.cparams[k], p.rparams[k])
    x = p.x[k]
    basic = (x > 0) & ~(np.isfinite(u) & (x == u))
    col = np.where(basic, 1, np.where(np.isfinite(u) & (x == u) & (x > 0), 2, 0)).astype(np.int8)
    return col, np.zeros(p.t.m, bool)


def planted_at_u(p):
    """x* of every LP with its nonbasic columns at 0 that have a finite upper bound moved to that bound, in index order, each one as
    long as the planted basis stays primal feasible with a margin (so that only bound flips lead back to x*).  The crossover's crash
    takes the planted basis (the only columns inside their bounds); the moved columns then have the wrong reduced cost."""
    x = p.x.copy()
    for k in range(len(x)):
        col, _ = planted_basis(p, k)
        _, b, u, _ = p.t.instantiate(p.cparams[k], p.rparams[k])
        A = p.t.matrix(p.rparams[k]).tocsc()
        basic = np.flatnonzero(col == 1)
        Binv = np.linalg.inv(A[:, basic].toarray())
        ub = u[basic]
        for j in np.flatnonzero((col == 0) & np.isfinite(u)):
            trial = x[k].copy()
            trial[j] = u[j]
            nb = np.setdiff1d(np.arange(p.t.n), basic)
            xb = Binv @ (b - A[:, nb] @ trial[nb])
            if (xb > 0.05 * np.where(np.isfinite(ub), ub, 1.0)).all() and (np.where(np.isfinite(ub), ub - xb, 1.0) > 0.05 * np.where(
                    np.isfinite(ub), ub, 1.0)).all():
                trial[basic] = xb
                x[k] = trial
    return x


def planted_third_basic_zero(p):
    """x* of every LP with every third of its basic columns (by index) set to 0"""
    x = p.x.copy()
    for k in range(len(x)):
        col, _ = planted_basis(p, k)
        b = np.flatnonzero(col == 1)
        x[k, b[::3]] = 0.0
    return x


def planted_inputs(p, x):
    return Inputs(p.t, p.cparams, p.rparams, np.zeros(len(p.x), np.int32), np.ascontiguousarray(x), p.y.copy())


def assignment_uniform(k, N, hi, seed=0):
    """the assignment LPs started from x = 1/k everywhere (every column inside its bounds): the crash fills the basis and the push
    moves the other k^2 - 2k + 1 columns onto a bound, most of them by a pivot"""
    I = assignment(k, N, hi, "zero", seed)
    I.x[:] = 1.0 / k
    return I


# ---------------------------------------------------------------------------------------------------------------------
# the cases: name -> (inputs, status every LP ends with, {trace path: floor of its count summed over the batch}).  The floors
# pin the paths each case exists to drive (tests/emu/harness_crossover.TRACE); they are floors, not counts.
# ---------------------------------------------------------------------------------------------------------------------
ROWS = {
    "assign40_zero_cost3": (lambda: assignment(40, 3, 3, "zero"), 0,
                            dict(dual_pivot=1, bland=1, cleanup_reinvert=1, artificial_out=1, redundant_row=3)),
    "assign40_zero_cost1000": (lambda: assignment(40, 3, 1000, "zero"), 0, dict(dual_pivot=1, cleanup_reinvert=1, redundant_row=3)),
    "assign40_identity_cost3": (lambda: assignment(40, 3, 3, "identity"), 0,
                                dict(primal_degenerate=1, bound_flip=1, cleanup_reinvert=1, artificial_out=1, redundant_row=3)),
    "assign40_identity_cost1000": (lambda: assignment(40, 3, 1000, "identity"), 0,
                                   dict(primal_degenerate=1, bland=1, bound_flip=1, cleanup_reinvert=1)),
    "assign60_identity_cost5": (lambda: assignment(60, 3, 5, "identity"), 0, dict(primal_degenerate=1, bland=1, cleanup_reinvert=1)),
    "assign40_uniform_cost1000": (lambda: assignment_uniform(40, 3, 1000), 0, dict(push_pivot=1, push_reinvert=1, redundant_row=3)),
    "planted40_at_u": (lambda: planted_inputs(planted40(), planted_at_u(planted40())), 0, dict(bound_flip=1)),
    "planted40_basic_third_zero": (lambda: planted_inputs(planted40(), planted_third_basic_zero(planted40())), 2, dict(round=3)),
}
ASSIGNMENT_K = {name: int(name[6:8]) for name in ROWS if name.startswith("assign")}

_p40 = []


def planted40():
    """the planted LPs of the planted40_* cases (m = 40, half bandwidth 3, N = 3)"""
    if not _p40:
        _p40.append(PL.planted(40, 3, N=3, bounded="mixed"))
    return _p40[0]


def check_basis_exact(I, v, k):
    """LP k's basis verifies as an exact optimum as it is; its x and objective are that optimum's"""
    basis = (v["col_status"][k].astype(np.int8), v["row_basic"][k].astype(bool))
    assert set(np.unique(basis[0])) <= {0, 1, 2}
    assert (basis[0] == 1).sum() + basis[1].sum() == I.t.m
    e = E.exact_optimum(I.t, I.cparams[k], I.rparams[k] if I.rparams is not None else None, basis=basis)
    assert np.abs(v["x"][k] - e.x).max() <= 1e-9 * max(1.0, np.abs(e.x).max())
    assert abs(v["obj"][k] - e.obj) <= 1e-9 * max(1.0, abs(e.obj))
    return e


# ---------------------------------------------------------------------------------------------------------------------
# the crossover's placement (csrc/dsp_lp.cu, xo_grid): the LP's work region in dynamic shared memory when
# xo::work_doubles(m, n, nnz) * 8 + sizeof(xo::Shared) fits in the device's opt-in shared memory per block, else in the workspace
# ---------------------------------------------------------------------------------------------------------------------
def work_doubles(m, n, nnz):
    """xo::work_doubles: the doubles of one LP's work region"""
    d = m * m + nnz + 4 * n + (n + m) + 7 * m
    i = 3 * m + 2 * n
    return (d + (i + 1) // 2 + 1) // 2 * 2


def shared_bytes():
    """sizeof(xo::Shared): two double and one int array of XO_THREADS entries, two doubles, an int and int[4], 8-byte aligned"""
    size = 2 * XO_THREADS * 8 + XO_THREADS * 4 + 2 * 8 + 4 + 4 * 4
    return (size + 7) // 8 * 8


def in_shared_memory(m, n, nnz, smem_optin=PL.H100_SMEM_OPTIN):
    return work_doubles(m, n, nnz) * 8 + shared_bytes() <= smem_optin


def planted_nnz(m, w, extra=0):
    """the nonzeros of planted(m, w, extra=0): an owned column per row spanning min(w, 2) + 1 rows and a coupling column spanning
    w + 1 rows, both cut off at the last row"""
    assert extra == 0
    we = min(w, m - 1)
    return sum(min(m - i, min(we, 2) + 1) + min(m - i, we + 1) for i in range(m))


def planted_boundary_m(w, smem_optin=PL.H100_SMEM_OPTIN):
    """the largest m whose planted(m, w, extra=0) crossover work region fits in shared memory (m + 1 does not)"""
    m = 1
    while in_shared_memory(m + 1, 2 * (m + 1), planted_nnz(m + 1, w), smem_optin):
        m += 1
    return m
