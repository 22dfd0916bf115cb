"""Exact optima and KKT residuals of template LPs (test infrastructure, no GPU).

    min c'x + k   s.t.  A x = b,  0 <= x <= u

``exact_optimum`` takes the LP exactly as a kernel receives it (``t.instantiate`` in binary64, every number converted to
``fractions.Fraction`` without rounding), lets HiGHS simplex find an optimal basis, takes that final basis (which columns and row
slacks are basic, which columns sit at 0 or at u), re-solves B x_B = b - N x_N and B'y = c_B in exact rational arithmetic and
verifies the KKT conditions exactly.  A basic row slack is a unit column whose value must come out exactly 0 (the rows are
equalities) and whose reduced cost forces y_i = 0.  Taking the basis from HiGHS rather than guessing it from x is what certifies
degenerate vertices: the dispatch LPs have zero prices, idle empty batteries and zero capacity factors, so fewer than m columns lie
strictly inside their bounds at almost every optimum.  The answer is the optimum of that very LP, not another solver's
approximation of it; when the basis does not verify, it raises (there is no fall-back to the floating-point answer).  The optimum
is unique in x when every nonbasic reduced cost is nonzero, and unique in y when every basic column lies strictly inside its bounds
(and no row slack is basic).  Either way, ``fixed`` marks the columns every optimal x has at the bound x* sits at (r*_j != 0,
complementary slackness with y*) and ``inside`` the columns at which every optimal y has a zero reduced cost (0 < x*_j < u_j).

``kkt_residuals`` measures any (x, y) a kernel returns -- degenerate LPs included -- against the same LP: primal residual, bound
violation, dual infeasibility of the unbounded columns (no artificial box) and the duality gap, with exactly rounded sums.
"""
from __future__ import annotations

import dataclasses
import math
from fractions import Fraction

import numpy as np

from oracle.highs import TIGHT


class NotCertified(AssertionError):
    """the HiGHS basis could not be verified as an exact optimum (singular, or a column or row misclassified)"""


@dataclasses.dataclass
class ExactOptimum:
    x: np.ndarray              # [n] x*, rounded from the exact value
    y: np.ndarray              # [m] y*
    obj: float                 # c'x* + k, rounded from the exact value
    lp_mag: float              # sum_j |c_j x*_j|
    basic: np.ndarray          # [n] bool
    unique_x: bool             # every nonbasic reduced cost is nonzero
    unique_y: bool             # every basic column lies strictly inside its bounds and no row slack is basic
    x_margin: float            # smallest distance of a basic x_j to its bounds, relative to max(1, |x*|_inf)
    r_margin: float            # smallest |r_j| of a nonbasic column, relative to |c|_inf
    r: np.ndarray = None       # [n] r* = c - A'y*, rounded from the exact value
    fixed: np.ndarray = None   # [n] bool, r*_j != 0: every optimal x has x_j at the bound x*_j sits at
    inside: np.ndarray = None  # [n] bool, 0 < x*_j < u_j: every optimal y has r_j(y) = 0


def _fr(v):
    return [Fraction(float(a)) for a in v]


def _solve_sparse(rows, rhs, nvar):
    """exact solution of a square sparse system: rows[e] = {var: Fraction}, rhs[e] = Fraction.  Variables are eliminated in the
    order of the first equation they appear in (time order for the stage templates), each from the shortest remaining equation
    that holds it, so the fill stays inside the band of a banded system."""
    rows = [dict(r) for r in rows]
    rhs = list(rhs)
    holders = [set() for _ in range(nvar)]
    for e, r in enumerate(rows):
        for v in r:
            holders[v].add(e)
    first = [min(h) if h else -1 for h in holders]
    if min(first, default=0) < 0 or len(rows) != nvar:
        raise NotCertified("singular basis (a variable in no equation, or not square)")
    done = [False] * len(rows)
    pivots = []
    for v in sorted(range(nvar), key=lambda v: first[v]):
        cands = [e for e in holders[v] if not done[e]]
        if not cands:
            raise NotCertified("singular basis")
        e = min(cands, key=lambda e: (len(rows[e]), e))
        done[e] = True
        pivots.append((v, e))
        prow, pv = rows[e], rows[e][v]
        for e2 in cands:
            if e2 == e:
                continue
            r2 = rows[e2]
            f = r2[v] / pv
            for v2, a in prow.items():
                nv = r2.get(v2, 0) - f * a
                if nv == 0:
                    if v2 in r2:
                        del r2[v2]
                        holders[v2].discard(e2)
                else:
                    r2[v2] = nv
                    holders[v2].add(e2)
            rhs[e2] -= f * rhs[e]
    sol = [Fraction(0)] * nvar
    for v, e in reversed(pivots):
        prow = rows[e]
        s = rhs[e]
        for v2, a in prow.items():
            if v2 != v:
                s -= a * sol[v2]
        sol[v] = s / prow[v]
    return sol


def _objective_constant(t, cp, rp):
    k = Fraction(float(t.o0))
    if t.Pr:
        k += sum((Fraction(float(a)) * Fraction(float(b)) for a, b in zip(t.omap, rp) if a != 0.0 and b != 0.0), Fraction(0))
    if t.Pc:
        k += sum((Fraction(float(a)) * Fraction(float(b)) for a, b in zip(t.ocmap, cp) if a != 0.0 and b != 0.0), Fraction(0))
    return k


def highs_basis(c, A, b, u):
    """HiGHS simplex (tolerances oracle.highs.TIGHT) on  min c'x  s.t.  A x = b, 0 <= x <= u  (A scipy CSC): its final basis as
    (col [n] int8: 0 at 0, 1 basic, 2 at u;  row_basic [m] bool: the row's slack is basic).  scipy's linprog returns x but not
    the basis, so this reads it through scipy's bundled HiGHS binding, which is private: it fails loudly where that is missing."""
    from scipy.optimize._highspy import _core as hc
    m, n = A.shape
    lp = hc.HighsLp()
    lp.num_col_, lp.num_row_ = n, m
    lp.col_cost_ = np.asarray(c, float)
    lp.col_lower_ = np.zeros(n)
    lp.col_upper_ = np.where(np.isfinite(u), u, hc.kHighsInf)
    lp.row_lower_ = lp.row_upper_ = np.asarray(b, float)
    mat = lp.a_matrix_
    mat.format_, mat.num_col_, mat.num_row_ = hc.MatrixFormat.kColwise, n, m
    mat.start_, mat.index_, mat.value_ = A.indptr, A.indices, A.data
    lp.a_matrix_ = mat
    h = hc._Highs()
    for k, v in dict(output_flag=False, solver="simplex", simplex_strategy=1, **TIGHT).items():      # (1: dual simplex)
        h.setOptionValue(k, v)
    if h.passModel(lp) != hc.HighsStatus.kOk or h.run() != hc.HighsStatus.kOk:
        raise NotCertified("HiGHS failed")
    if h.getModelStatus() != hc.HighsModelStatus.kOptimal:
        raise NotCertified(f"HiGHS: {h.modelStatusToString(h.getModelStatus())}")
    bs = h.getBasis()
    if not bs.valid:
        raise NotCertified("HiGHS returned no valid basis")
    code = {hc.HighsBasisStatus.kLower: 0, hc.HighsBasisStatus.kBasic: 1, hc.HighsBasisStatus.kUpper: 2}
    col = np.array([code.get(v, -1) for v in bs.col_status], np.int8)
    if (col < 0).any():
        raise NotCertified("HiGHS basis has a column neither basic nor at a bound")
    return col, np.array([v == hc.HighsBasisStatus.kBasic for v in bs.row_status])


def exact_optimum(t, cparams_row, rparams_row, basis=None) -> ExactOptimum:
    """the exact optimum of one LP of template t (see the module docstring); raises NotCertified when HiGHS' final basis -- or
    ``basis``, a (col, row_basic) pair as highs_basis returns it -- does not verify in exact arithmetic"""
    cp = np.asarray(cparams_row, float)
    rp = np.asarray(rparams_row if rparams_row is not None else np.zeros(0), float)
    c, b, u, _ = t.instantiate(cp, rp)
    A = t.matrix(rp).tocsc(copy=True)
    A.sort_indices()
    m, n = A.shape
    fin = np.isfinite(u)
    col, row_basic = highs_basis(c, A, b, u) if basis is None else basis
    basic, at_hi = col == 1, col == 2
    at_lo = col == 0
    if (at_hi & ~fin).any():
        raise NotCertified("an unbounded column at its upper bound")
    if basic.sum() + row_basic.sum() != m:
        raise NotCertified(f"{int(basic.sum())} basic columns and {int(row_basic.sum())} basic row slacks for {m} rows")
    # exact data
    cF, bF = _fr(c), _fr(b)
    uF = [Fraction(float(v)) if f else None for v, f in zip(u, fin)]
    cols = [(A.indices[A.indptr[j]:A.indptr[j + 1]], _fr(A.data[A.indptr[j]:A.indptr[j + 1]])) for j in range(n)]
    xF = [Fraction(0)] * n
    for j in np.flatnonzero(at_hi):
        xF[j] = uF[j]
    rhs = list(bF)
    for j in np.flatnonzero(at_hi):
        for i, a in zip(*cols[j]):
            rhs[i] -= a * xF[j]
    bidx = np.flatnonzero(basic)
    sidx = np.flatnonzero(row_basic)
    pos = {j: k for k, j in enumerate(bidx)}
    rowsB = [dict() for _ in range(m)]                 # B x_B = rhs: equation i, variable pos[j]; then the basic row slacks
    for j in bidx:
        for i, a in zip(*cols[j]):
            rowsB[i][pos[j]] = a
    for k, i in enumerate(sidx):
        rowsB[i][len(bidx) + k] = Fraction(1)
    xB = _solve_sparse(rowsB, rhs, m)
    for j, v in zip(bidx, xB):
        xF[j] = v
    if any(xB[len(bidx):]):
        raise NotCertified("a basic row slack is nonzero")
    rowsT = [{int(i): a for i, a in zip(*cols[j])} for j in bidx] + [{int(i): Fraction(1)} for i in sidx]   # B'y = c_B
    yF = _solve_sparse(rowsT, [cF[j] for j in bidx] + [Fraction(0)] * len(sidx), m)
    # exact KKT
    rF = []
    for j in range(n):
        s = cF[j]
        for i, a in zip(*cols[j]):
            s -= a * yF[i]
        rF.append(s)
    Ax = [Fraction(0)] * m
    for j in range(n):
        if xF[j]:
            for i, a in zip(*cols[j]):
                Ax[i] += a * xF[j]
    if any(Ax[i] != bF[i] for i in range(m)):
        raise NotCertified("A x != b")
    for j in range(n):
        if xF[j] < 0 or (fin[j] and xF[j] > uF[j]):
            raise NotCertified(f"column {j} outside its bounds")
        if basic[j] and rF[j] != 0:
            raise NotCertified(f"basic column {j} has a nonzero reduced cost")
        if at_lo[j] and rF[j] < 0:
            raise NotCertified(f"column {j} at 0 with a negative reduced cost")
        if at_hi[j] and rF[j] > 0:
            raise NotCertified(f"column {j} at its bound with a positive reduced cost")
    objF = sum((cF[j] * xF[j] for j in range(n) if xF[j]), Fraction(0)) + _objective_constant(t, cp, rp)
    inside = [min(xF[j], uF[j] - xF[j]) if fin[j] else xF[j] for j in bidx]
    sc = max(1e-300, float(np.abs(c).max(initial=0.0)))
    x = np.array([float(v) for v in xF])
    return ExactOptimum(x=x, y=np.array([float(v) for v in yF]), obj=float(objF), lp_mag=math.fsum(np.abs(c * x)),
                        basic=basic, unique_x=all(rF[j] != 0 for j in range(n) if not basic[j]),
                        unique_y=all(v > 0 for v in inside) and not row_basic.any(),
                        x_margin=float(min(inside, default=math.inf)) / max(1.0, float(np.abs(x).max(initial=0.0))),
                        r_margin=float(min((abs(rF[j]) for j in range(n) if not basic[j]), default=math.inf)) / sc,
                        r=np.array([float(v) for v in rF]), fixed=np.array([v != 0 for v in rF]),
                        inside=np.array([xF[j] > 0 and (not fin[j] or xF[j] < uF[j]) for j in range(n)]))


def kkt_residuals(t, cparams_row, rparams_row, x, y, lp_zero=False):
    """KKT residuals of any (x, y) for one LP of template t, with exactly rounded sums (math.fsum):
      primal    |A x - b|_inf            relative to the primal scale max(1, |b|_inf, |u_finite|_inf)
      bound     largest violation of 0 <= x <= u, same scale
      dual_inf  max(-r_j, 0) over the UNBOUNDED columns (r = c - A'y; no box is put on them), relative to |c|_inf
      gap       |c'x - (b'y + sum_bounded u_j min(r_j, 0))|, relative to sum_j |c_j x_j| (>= |c'x|)
    A (x, y) that is primal feasible, dual feasible and has no gap is optimal, degenerate LP or not.

    An LP whose LP part is identically zero at the optimum -- c = 0, or ``lp_zero`` (the caller knows every priced column is 0
    at the optimum, ExactOptimum.lp_mag == 0) -- has y* = 0 among its optimal duals and a solver's y is rounding noise there, with
    nothing to measure it against: dual_inf and gap are None (not applicable) and only the primal measures are reported."""
    cp = np.asarray(cparams_row, float)
    rp = np.asarray(rparams_row if rparams_row is not None else np.zeros(0), float)
    c, b, u, _ = t.instantiate(cp, rp)
    A = t.matrix(rp)
    Ar, Ac = A.tocsr(), A.tocsc()
    x = np.asarray(x, float); y = np.asarray(y, float)
    m, n = A.shape
    fin = np.isfinite(u)
    sb = max(1.0, float(np.abs(b).max(initial=0.0)), float(np.abs(u[fin]).max(initial=0.0)))
    ax = [math.fsum(list(Ar.data[Ar.indptr[i]:Ar.indptr[i + 1]] * x[Ar.indices[Ar.indptr[i]:Ar.indptr[i + 1]]]) + [-b[i]])
          for i in range(m)]
    out = dict(primal=float(np.abs(ax).max(initial=0.0)) / sb,
               bound=max(0.0, -float(x.min(initial=0.0)), float(np.max((x - u)[fin], initial=0.0))) / sb)
    sc = float(np.abs(c).max(initial=0.0))
    mag = math.fsum(np.abs(c * x))
    if lp_zero or sc == 0.0:
        return dict(out, dual_inf=None, gap=None)
    r = np.array([math.fsum([c[j]] + list(-Ac.data[Ac.indptr[j]:Ac.indptr[j + 1]] * y[Ac.indices[Ac.indptr[j]:Ac.indptr[j + 1]]]))
                  for j in range(n)])
    primal_obj = math.fsum(c * x)
    ur = u[fin] * np.minimum(r[fin], 0.0)
    dual_obj = math.fsum(list(b * y) + list(ur))
    return dict(out, dual_inf=float(np.max(-r[~fin], initial=0.0)) / sc if (~fin).any() else 0.0,
                gap=abs(primal_obj - dual_obj) / mag if mag > 0.0 else (0.0 if primal_obj == dual_obj else math.inf))
