"""Exact ranging of template LPs over a given basis (test infrastructure, no GPU): the interval of theta over which a basis stays
optimal along a direction of the batch parameters, by the rules of dsp_lp_ranging (include/dsp_lp.h), in rational arithmetic on the
LP as the kernels receive it; and the exact check of a basis at moved parameters.  Builds on exact_lp's exact basic solutions."""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

import exact_lp as E

FEAS = 1e-9      # the ranging's on-bound tolerance (relative to the primal / dual scale)
RATE = 1e-9      # and its negligible-rate threshold (relative to the direction's scale)


def _lp(t, cp, rp):
    cp = np.asarray(cp, float)
    rp = np.asarray(rp if rp is not None else np.zeros(0), float)
    c, b, u, _ = t.instantiate(cp, rp)
    A = t.matrix(rp).tocsc(copy=True)
    A.sort_indices()
    cols = [(A.indices[A.indptr[j]:A.indptr[j + 1]], E._fr(A.data[A.indptr[j]:A.indptr[j + 1]])) for j in range(t.n)]
    return cp, rp, c, b, np.maximum(u, 0.0), cols


def verify(t, cp, rp, basis):
    """the exact objective c'x + k of the basis' basic solution at (cp, rp) when the basis is optimal there in exact arithmetic; raises
    exact_lp.NotCertified otherwise.  A column with u = 0 may sit at either bound whatever the sign of its reduced cost."""
    cp, rp, c, b, u, cols = _lp(t, cp, rp)
    col, rb = np.asarray(basis[0]), np.asarray(basis[1]).astype(bool)
    fin = np.isfinite(u)
    if (col == 2)[~fin].any() or (col == 1).sum() + rb.sum() != t.m:
        raise E.NotCertified("not a basis")
    uF = [Fraction(float(v)) if f else None for v, f in zip(u, fin)]
    xF, sF, yF, rF = E._vertex(cols, E._fr(c), E._fr(b), uF, col, rb)
    if any(sF.values()):
        raise E.NotCertified("a basic artificial is nonzero")
    for j in range(t.n):
        if xF[j] < 0 or (fin[j] and xF[j] > uF[j]):
            raise E.NotCertified(f"column {j} outside its bounds")
        if col[j] != 1 and not (fin[j] and uF[j] == 0):
            if (col[j] == 0 and rF[j] < 0) or (col[j] == 2 and rF[j] > 0):
                raise E.NotCertified(f"column {j}: reduced cost of the wrong sign")
    return sum((Fraction(float(c[j])) * xF[j] for j in range(t.n) if xF[j]), Fraction(0)) + E._objective_constant(t, cp, rp)


def _dot(M, g):
    """M @ g exactly (M a dense or scipy matrix of floats, g floats) as Fractions"""
    M = M.toarray() if hasattr(M, "toarray") else np.asarray(M)
    out = []
    for row in np.atleast_2d(M):
        nz = np.flatnonzero(row)
        out.append(sum((Fraction(float(row[q])) * Fraction(float(g[q])) for q in nz if g[q] != 0.0), Fraction(0)))
    return out


def exact_range(t, cp, rp, basis, dir_c, dir_r):
    """(lo, hi) of the basis along (dir_c [Pc], dir_r [Pr]) by dsp_lp_ranging's rules in exact arithmetic (floats; +-inf where
    unbounded).  The on-bound tolerances and rate thresholds are the kernel's, taken at their floating-point values."""
    cp, rp, c, b, u, cols = _lp(t, cp, rp)
    col, rb = np.asarray(basis[0]), np.asarray(basis[1]).astype(bool)
    n, m = t.n, t.m
    fin = np.isfinite(u)
    uF = [Fraction(float(v)) if f else None for v, f in zip(u, fin)]
    xF, sF, yF, rF = E._vertex(cols, E._fr(c), E._fr(b), uF, col, rb)
    gc = np.zeros(t.Pc) if dir_c is None else np.asarray(dir_c, float)
    gr = np.zeros(t.Pr) if dir_r is None else np.asarray(dir_r, float)
    dc = _dot(t.Cmap, gc) if t.Pc else [Fraction(0)] * n
    db = _dot(t.Bmap, gr) if t.Pr else [Fraction(0)] * m
    du = _dot(t.Umap, gr) if t.Pr else [Fraction(0)] * n
    du = [d if f else Fraction(0) for d, f in zip(du, fin)]
    dxF, dsF, dyF, ddF = E._vertex(cols, dc, db, du, col, rb)
    tolp = Fraction(FEAS * max(1.0, float(np.abs(b).max(initial=0.0)), float(np.abs(u[fin]).max(initial=0.0))))
    told = Fraction(FEAS * (float(np.abs(c).max(initial=0.0)) or 1.0))
    rtp = Fraction(RATE * float(max(max((abs(v) for v in db), default=0), max((abs(v) for v in du), default=0))))
    rtd = Fraction(RATE * float(max((abs(v) for v in dc), default=0)))
    hi = lo = None                                       # None: unbounded

    def block(g, dg, tol, rt):
        nonlocal hi, lo
        if not abs(dg) > rt:
            return
        r = Fraction(0) if g <= tol else g / abs(dg)
        if dg < 0:
            hi = r if hi is None else min(hi, r)
        else:
            lo = r if lo is None else min(lo, r)

    for i in np.flatnonzero(rb):
        if abs(dsF[int(i)]) > rtp:
            hi = lo = Fraction(0)
    for j in range(n):
        if col[j] == 1:
            block(xF[j], dxF[j], tolp, rtp)
            if fin[j]:
                block(uF[j] - xF[j], du[j] - dxF[j], tolp, rtp)
            continue
        if col[j] == 2:
            block(uF[j], du[j], tolp, rtp)
        if fin[j] and uF[j] == 0:
            if du[j] == 0:
                continue
            if (rF[j] if col[j] == 0 else -rF[j]) < -told:            # fixed, at the wrong bound for its reduced cost
                if du[j] > 0:
                    hi = Fraction(0)
                else:
                    lo = Fraction(0)
                continue
        if col[j] == 0:
            block(rF[j], ddF[j], told, rtd)
        else:
            block(-rF[j], -ddF[j], told, rtd)
    return (-math.inf if lo is None else -float(lo)), (math.inf if hi is None else float(hi))


def moved(t, cp, rp, dir_c, dir_r, theta):
    """the parameters at theta along the direction (floating point, as a caller would form them)"""
    cp2 = np.asarray(cp, float) + (theta * np.asarray(dir_c, float) if dir_c is not None and t.Pc else 0.0)
    rp2 = None if rp is None else np.asarray(rp, float) + (theta * np.asarray(dir_r, float) if dir_r is not None and t.Pr else 0.0)
    return cp2, rp2
