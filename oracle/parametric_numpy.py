"""numpy mirror of the parametric walk (dsp_lp_parametric, dispatches_b200/csrc/dsp_parametric.cuh, DESIGN.md 4.8).

An independent implementation of the same rules on one LP of a template and a basis optimal at theta = 0 (col_status [n]: 0 at 0,
1 basic, 2 at u; row_basic [m]): along one direction (dir_c, dir_r) of the batch parameters, the event log of basis changes and bound
flips up to theta_end.  The linear algebra is different on purpose: at every event the LP is formed afresh at theta (p + theta dir, in
numpy) and its basis factorised from scratch (scipy.linalg.lu_factor), with LU solves for x_B, y, the direction's rates, the pivot
column and the pivot row; no explicit inverse, no product-form update, no iterative refinement.  The ranging step is
oracle/ranging_numpy.py's rules with the blocking entry kept; the crossover's pivot tolerance (oracle/crossover_numpy.py) is 1e-7.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sl

from . import ranging_numpy as RN

PIVOT = 1e-7
BLAND_AFTER = 50
OPTIMAL, MAX_ITER, NUMERICAL, INFEASIBLE, UNBOUNDED = 0, 1, 2, 3, 4
BASIC_LO, BASIC_UP, ARTIFICIAL, BOUND, DUAL, UNFIX = range(6)


class _LP:
    """the LP at theta with the basis factorised: x (columns and artificials), y, d, the tolerances; pinf / dinf: primal / dual
    infeasible beyond them"""

    def __init__(self, t, cp, rp, cs, rb):
        c, b, u, _ = t.instantiate(cp, rp)
        self.A = np.asarray(t.matrix(rp).toarray(), float)
        self.b, self.c, self.u = np.asarray(b, float), np.asarray(c, float), np.maximum(np.asarray(u, float), 0.0)
        m, n = self.A.shape
        fin = np.isfinite(self.u)
        self.tolp = RN.FEAS * max(1.0, np.abs(self.b).max(initial=0.0), np.abs(self.u[fin]).max(initial=0.0))
        self.told = RN.FEAS * (np.abs(self.c).max(initial=0.0) or 1.0)
        self.cs, self.rb = cs.copy(), rb.copy()
        self.head = list(np.flatnonzero(cs == 1)) + [n + i for i in np.flatnonzero(rb == 1)]
        self.ok = len(self.head) == m and not ((cs == 2) & ~fin).any()
        if not self.ok:
            return
        self.Ae = np.hstack([self.A, np.eye(m)])
        B = self.Ae[:, self.head]
        with np.errstate(all="ignore"):
            self.lu = sl.lu_factor(B)
        if not np.all(np.isfinite(self.lu[0])) or (np.abs(np.diag(self.lu[0])) <= 1e-12 * np.abs(B).max(0)).any():
            self.ok = False
            return
        self.xe = np.concatenate([np.where(cs == 2, self.u, 0.0), np.zeros(m)])
        self.xe[self.head] = sl.lu_solve(self.lu, self.b - self.A @ self.xe[:n])
        cb = np.array([self.c[h] if h < n else 0.0 for h in self.head])
        self.y = sl.lu_solve(self.lu, cb, trans=1)
        self.d = self.c - self.A.T @ self.y
        ub = np.concatenate([self.u, np.zeros(m)])[self.head]
        xb = self.xe[self.head]
        self.pinf = bool(((xb < -self.tolp) | (xb > ub + self.tolp)).any())
        nb = (cs != 1) & (self.u > 0.0)
        self.dinf = bool((nb & (((cs == 0) & (self.d < -self.told)) | ((cs == 2) & (self.d > self.told)))).any())

    def upper(self, v):
        return self.u[v] if v < len(self.u) else 0.0


def _segment(L, dc, db, du, dk):
    """the ranging step with the blocking entry of the upper side: (hi, (var, kind) or None, dobj, d2obj, dxb, dd)"""
    A, n = L.A, L.A.shape[1]
    fin = np.isfinite(L.u)
    du = np.where(fin, du, 0.0)
    dcb = np.array([dc[h] if h < n else 0.0 for h in L.head])
    dd = dc - A.T @ sl.lu_solve(L.lu, dcb, trans=1)
    dxn = np.where(L.cs == 2, du, 0.0)
    dxb = sl.lu_solve(L.lu, db - A @ dxn)
    rtp = RN.RATE * max(np.abs(db).max(initial=0.0), np.abs(du).max(initial=0.0))
    rtd = RN.RATE * np.abs(dc).max(initial=0.0)
    best = [np.inf, 0.0, np.inf]                          # (ratio, class, var * 8 + kind)

    def keep(r, cls, v, kind):
        key = [r, cls, v * 8 + kind]
        if key < best:
            best[:] = key

    def block(g, dg, tol, rt, cls, v, kind):
        if abs(dg) > rt and dg < 0:
            keep(0.0 if g <= tol else g / abs(dg), cls, v, kind)

    for k, v in enumerate(L.head):
        x, g = L.xe[v], dxb[k]
        if v >= n:
            if abs(g) > rtp:
                keep(0.0, 0.0, v, ARTIFICIAL)
            continue
        block(x, g, L.tolp, rtp, 0.0, v, BASIC_LO)
        if fin[v]:
            block(L.u[v] - x, du[v] - g, L.tolp, rtp, 0.0, v, BASIC_UP)
    for j in range(n):
        if L.cs[j] == 1:
            continue
        if L.cs[j] == 2:
            block(L.u[j], du[j], L.tolp, rtp, 0.0, j, BOUND)
        if L.u[j] <= 0.0:
            if du[j] == 0.0:
                continue
            if (L.d[j] if L.cs[j] == 0 else -L.d[j]) < -L.told:
                if du[j] > 0:
                    keep(0.0, -1.0, j, UNFIX)
                continue
        if L.cs[j] == 0:
            block(L.d[j], dd[j], L.told, rtd, 1.0, j, DUAL)
        else:
            block(-L.d[j], -dd[j], L.told, rtd, 1.0, j, DUAL)
    dx = dxn.copy()
    for k, v in enumerate(L.head):
        if v < n:
            dx[v] = dxb[k]
    dobj = float(dc @ L.xe[:n] + L.c @ dx + dk)
    blk = None if np.isinf(best[0]) else (int(best[2]) // 8, int(best[2]) % 8)
    return best[0], blk, dobj, float(2.0 * dc @ dx), dxb, dd


def walk(t, cparams, rparams, col_status, row_basic, dir_c, dir_r, theta_end=np.inf, S=256):
    """dict(theta, obj, dobj, d2obj, enter, leave, leave_to [S], count, status) of one LP of template t along (dir_c [Pc], dir_r [Pr])"""
    cp0 = np.asarray(cparams, float).reshape(t.Pc)
    rp0 = np.asarray(rparams if rparams is not None else np.zeros(0), float).reshape(t.Pr)
    gc = np.zeros(t.Pc) if dir_c is None or not t.Pc else np.asarray(dir_c, float)
    gr = np.zeros(t.Pr) if dir_r is None or not t.Pr else np.asarray(dir_r, float)
    out = dict(theta=np.full(S, np.nan), obj=np.full(S, np.nan), dobj=np.full(S, np.nan), d2obj=np.full(S, np.nan),
               enter=np.full(S, -1, np.int32), leave=np.full(S, -1, np.int32), leave_to=np.full(S, -1, np.int8), count=0, status=NUMERICAL)
    in_A = np.zeros(t.Pr, bool)
    if t.amap is not None:
        in_A[np.asarray(t.amap[2], int)] = True
    if (gr[in_A] != 0.0).any():
        return out
    n = t.n
    dc = t.Cmap @ gc if t.Pc else np.zeros(n)
    db = t.Bmap @ gr if t.Pr else np.zeros(t.m)
    du = t.Umap @ gr if t.Pr else np.zeros(n)
    dk = (float(t.omap @ gr) if t.Pr else 0.0) + (float(t.ocmap @ gc) if t.Pc else 0.0)
    at = lambda th: (cp0 + th * gc, rp0 + th * gr) if th != 0.0 else (cp0, rp0)
    cs, rb = np.asarray(col_status, np.int8).copy(), np.asarray(row_basic, np.int8).copy()
    th = 0.0
    L = _LP(t, *at(th), cs, rb)
    if not L.ok or L.pinf or L.dinf:
        return out
    cnt, status, ev, degen = 0, OPTIMAL, (-1, -1, -1), 0

    def objective(L, th):
        cp, rp = at(th)
        o = float(t.o0) + (float(t.omap @ rp) if t.Pr else 0.0) + (float(t.ocmap @ cp) if t.Pc else 0.0)
        return float(L.c @ L.xe[:n]) + o

    def record(e, th, obj, d1, d2, ev):
        out["theta"][e], out["obj"][e], out["dobj"][e], out["d2obj"][e] = th, obj, d1, d2
        out["enter"][e], out["leave"][e], out["leave_to"][e] = ev

    while True:
        hi, blk, d1, d2, dxb, dd = _segment(L, dc, db, du, dk)
        record(cnt, th, objective(L, th), d1, d2, ev)
        cnt += 1
        tn = th + hi
        if blk is None or not tn < theta_end:
            break
        if cnt == S:
            status = MAX_ITER
            break
        degen = degen + 1 if tn == th else 0
        low_index = degen >= BLAND_AFTER
        v, kind = blk
        rate_art = dxb[L.head.index(v)] if kind == ARTIFICIAL else 0.0
        dx_old = {h: dxb[k] for k, h in enumerate(L.head)}
        th = tn
        L = _LP(t, *at(th), cs, rb)
        if not L.ok:
            status = NUMERICAL
            break
        ev = (-1, v, -1)
        if kind == BOUND:
            status = INFEASIBLE
        elif kind == UNFIX:
            up = L.d[v] < 0.0
            cs[v] = 2 if up else 0
            ev = (-1, v, 2 if up else 0)
        elif kind == DUAL:                                # primal simplex: v enters
            q, direction = v, (1 if cs[v] == 0 else -1)
            al = sl.lu_solve(L.lu, L.Ae[:, q])
            tol_piv = PIVOT * np.abs(al).max(initial=0.0)
            cands = []
            for r, h in enumerate(L.head):
                s_ = direction * al[r]
                if abs(s_) < tol_piv or s_ == 0.0:
                    continue
                x, up, dxu = L.xe[h], L.upper(h), dx_old.get(h, 0.0) if h < n else 0.0
                if s_ > 0:
                    gap, dgap = x, dxu
                elif up < np.inf:
                    gap, dgap = up - x, (du[h] - dxu if h < n else 0.0)
                else:
                    continue
                a = abs(s_)
                cands.append(((max(gap, 0.0) / a if h < n else 0.0), dgap / a, 0.0 if low_index else -a, h, r, s_ < 0))
            uq = L.u[q]
            if not cands and uq == np.inf:
                status = UNBOUNDED
            else:
                best = min(cands) if cands else None
                if best is None or uq < best[0] or (uq == best[0] and du[q] <= best[1]):
                    cs[q] = 2 if direction > 0 else 0
                    ev = (-1, q, 2 if direction > 0 else 0)
                else:
                    h, to_up = best[3], best[5]
                    cs[q] = 1
                    if h < n:
                        cs[h] = 2 if to_up else 0
                    else:
                        rb[h - n] = 0
                    ev = (q, h, 2 if to_up and h < n else 0)
        else:                                             # dual simplex: basic v leaves to the bound it reached
            r = L.head.index(v)
            below = kind == BASIC_LO or (kind == ARTIFICIAL and rate_art < 0.0)
            direction = -1 if below else 1
            er = np.zeros(t.m); er[r] = 1.0
            rho = sl.lu_solve(L.lu, er, trans=1)
            rmax = np.abs(rho).max(initial=0.0)
            cands = []
            for j in range(n):
                if cs[j] == 1 or not (L.u[j] > 0.0 or du[j] > 0.0):
                    continue
                col = L.A[:, j]
                a = float(rho @ col)
                if not abs(a) >= PIVOT * rmax * np.abs(col).max(initial=0.0) or a == 0.0:
                    continue
                lo = cs[j] == 0
                if not ((lo and a * direction > 0) or (not lo and a * direction < 0)):
                    continue
                slack = max(L.d[j], 0.0) if lo else max(-L.d[j], 0.0)
                cands.append((slack / abs(a), (dd[j] if lo else -dd[j]) / abs(a), 0.0 if low_index else -abs(a), j))
            if not cands:
                status = INFEASIBLE
            else:
                e = min(cands)[3]
                cs[e] = 1
                if v < n:
                    cs[v] = 0 if below else 2
                else:
                    rb[v - n] = 0
                ev = (e, v, 0 if below or v >= n else 2)
        if status != OPTIMAL:
            record(cnt, th, objective(L, th), np.nan, np.nan, (-1, -1, -1))
            cnt += 1
            break
        L = _LP(t, *at(th), cs, rb)
        if not L.ok:
            status = NUMERICAL
            break
        if L.pinf and L.dinf:
            status = NUMERICAL
            break
    out["count"], out["status"] = cnt, status
    return out
