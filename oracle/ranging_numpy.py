"""numpy mirror of the ranging post-pass (dsp_lp_ranging, dispatches_b200/csrc/dsp_ranging.cuh, DESIGN.md 4.7).

An independent implementation of the same rules on one LP  min c'x + k, A x = b, 0 <= x <= u  and a basis (col_status [n]: 0 at 0,
1 basic, 2 at u; row_basic [m]: the row's artificial, a unit column with bounds [0, 0], is basic): for each direction (dc, db, du, dk)
of the LP's data, the interval [lo, hi] of theta over which the basis stays optimal for (c + theta dc, b + theta db, u + theta du), and
dobj, d2obj of obj(theta) = obj + dobj theta + d2obj theta^2 / 2 inside it.  The linear algebra is different on purpose: one LU
factorisation of B (scipy.linalg.lu_factor) and LU solves, no explicit inverse and no iterative refinement.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sl

FEAS = 1e-9      # on-bound tolerance, relative to the primal scale max(1, |b|_inf, |u_finite|_inf) and to |c|_inf (the crossover's)
RATE = 1e-9      # a rate at most this, relative to the direction's scale, does not block
OPTIMAL, NUMERICAL = 0, 2


class Basis:
    """the LP at theta = 0 with its basis factorised: x, y, d; ``status`` NUMERICAL where the basis is not a feasible optimal one"""

    def __init__(self, A, b, c, u, col_status, row_basic):
        A = np.asarray(A.toarray() if hasattr(A, "toarray") else A, float)
        self.A, self.b, self.c = A, np.asarray(b, float), np.asarray(c, float)
        self.u = np.maximum(np.asarray(u, float), 0.0)
        m, n = A.shape
        cs, rb = np.asarray(col_status), np.asarray(row_basic)
        fin = np.isfinite(self.u)
        self.tolp = FEAS * max(1.0, np.abs(self.b).max(initial=0.0), np.abs(self.u[fin]).max(initial=0.0))
        self.told = FEAS * (np.abs(self.c).max(initial=0.0) or 1.0)
        self.cs, self.rb = cs, rb
        self.head = list(np.flatnonzero(cs == 1)) + [n + i for i in np.flatnonzero(rb == 1)]
        self.status = OPTIMAL
        if len(self.head) != m or not np.isin(cs, (0, 1, 2)).all() or not np.isin(rb, (0, 1)).all() or ((cs == 2) & ~fin).any():
            self.status = NUMERICAL
            return
        Ae = np.hstack([A, np.eye(m)])
        self.B = Ae[:, self.head]
        try:
            with np.errstate(all="ignore"):
                self.lu = sl.lu_factor(self.B, check_finite=True)
            if not np.all(np.isfinite(self.lu[0])) or (np.abs(np.diag(self.lu[0])) <= 1e-12 * np.abs(self.B).max(0)).any():
                raise np.linalg.LinAlgError
        except (np.linalg.LinAlgError, ValueError):
            self.status = NUMERICAL
            return
        self.at_up = cs == 2
        self.xn = np.where(self.at_up, self.u, 0.0)
        self.x = self.xn.copy()
        xb = sl.lu_solve(self.lu, self.b - A @ self.xn)
        self.xe = np.concatenate([self.x, np.zeros(m)])
        self.xe[self.head] = xb
        self.x = self.xe[:n]
        cb = np.array([self.c[h] if h < n else 0.0 for h in self.head])
        self.y = sl.lu_solve(self.lu, cb, trans=1)
        self.d = self.c - A.T @ self.y
        ub = np.concatenate([self.u, np.zeros(m)])[self.head]
        viol = (xb < -self.tolp) | (xb > ub + self.tolp)
        nb = (cs != 1) & (self.u > 0.0)
        dinf = nb & (((cs == 0) & (self.d < -self.told)) | ((cs == 2) & (self.d > self.told)))
        if viol.any() or dinf.any():
            self.status = NUMERICAL

    def range(self, dc, db, du, dk=0.0):
        """(lo, hi, dobj, d2obj) along the direction: dc [n], db [m], du [n] (ignored where u is infinite), dk the constant term's rate"""
        A, m, n = self.A, self.A.shape[0], self.A.shape[1]
        fin = np.isfinite(self.u)
        dc, db = np.asarray(dc, float), np.asarray(db, float)
        du = np.where(fin, np.asarray(du, float), 0.0)
        dcb = np.array([dc[h] if h < n else 0.0 for h in self.head])
        dy = sl.lu_solve(self.lu, dcb, trans=1)
        dd = dc - A.T @ dy
        dxn = np.where(self.at_up, du, 0.0)
        dxb = sl.lu_solve(self.lu, db - A @ dxn)
        rtp = RATE * max(np.abs(db).max(initial=0.0), np.abs(du).max(initial=0.0))
        rtd = RATE * np.abs(dc).max(initial=0.0)
        hi, lo = np.inf, np.inf

        def block(g, dg, tol, rt):
            nonlocal hi, lo
            if not abs(dg) > rt:
                return
            r = 0.0 if g <= tol else g / abs(dg)
            if dg < 0:
                hi = min(hi, r)
            else:
                lo = min(lo, r)

        for k, v in enumerate(self.head):
            x, g = self.xe[v], dxb[k]
            if v >= n:
                if abs(g) > rtp:
                    hi = lo = 0.0
                continue
            block(x, g, self.tolp, rtp)
            if fin[v]:
                block(self.u[v] - x, du[v] - g, self.tolp, rtp)
        for j in range(n):
            if self.cs[j] == 1:
                continue
            if self.cs[j] == 2:
                block(self.u[j], du[j], self.tolp, rtp)
            if self.u[j] <= 0.0:
                if du[j] == 0.0:
                    continue
                if (self.d[j] if self.cs[j] == 0 else -self.d[j]) < -self.told:      # fixed, at the wrong bound for its d_j
                    if du[j] > 0:
                        hi = 0.0
                    else:
                        lo = 0.0
                    continue
            if self.cs[j] == 0:
                block(self.d[j], dd[j], self.told, rtd)
            else:
                block(-self.d[j], -dd[j], self.told, rtd)
        dx = dxn.copy()
        for k, v in enumerate(self.head):
            if v < n:
                dx[v] = dxb[k]
        dobj = float(dc @ self.x + self.c @ dx + dk)
        return -lo if lo else 0.0, hi, dobj, float(2.0 * dc @ dx)


def ranging(t, cparams, rparams, col_status, row_basic, dir_c, dir_r):
    """dict(lo, hi, dobj, d2obj [K], status) of one LP of template t (cparams / rparams one row) along the directions dir_c [K,Pc] and
    dir_r [K,Pr] of its batch parameters (None: not moved); NaN where the LP's basis is not OPTIMAL, and in the columns of directions
    that move a parameter entering a matrix term"""
    cp = np.asarray(cparams, float).reshape(t.Pc)
    rp = np.asarray(rparams if rparams is not None else np.zeros(0), float).reshape(t.Pr)
    c, b, u, _ = t.instantiate(cp, rp)
    K = (dir_c if dir_c is not None else dir_r).shape[0]
    gc = np.zeros((K, t.Pc)) if dir_c is None or not t.Pc else np.asarray(dir_c, float)
    gr = np.zeros((K, t.Pr)) if dir_r is None or not t.Pr else np.asarray(dir_r, float)
    out = dict(lo=np.full(K, np.nan), hi=np.full(K, np.nan), dobj=np.full(K, np.nan), d2obj=np.full(K, np.nan))
    Bs = Basis(t.matrix(rp), b, c, u, col_status, row_basic)
    out["status"] = Bs.status
    if Bs.status != OPTIMAL:
        return out
    in_A = np.zeros(t.Pr, bool)
    if t.amap is not None:
        in_A[np.asarray(t.amap[2], int)] = True
    for k in range(K):
        if (gr[k][in_A] != 0.0).any():
            continue
        dk = (float(t.omap @ gr[k]) if t.Pr else 0.0) + (float(t.ocmap @ gc[k]) if t.Pc else 0.0)
        r = Bs.range(t.Cmap @ gc[k] if t.Pc else np.zeros(t.n), t.Bmap @ gr[k] if t.Pr else np.zeros(t.m),
                     t.Umap @ gr[k] if t.Pr else np.zeros(t.n), dk)
        out["lo"][k], out["hi"][k], out["dobj"][k], out["d2obj"][k] = r
    return out
