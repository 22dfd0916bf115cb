"""CPU ORACLE (test infrastructure -- NOT product code).

Batched numpy mirror of the dense kernel (dispatches_b200/csrc/dsp_lp.cu, dsp_ipm_dense_kernel; DESIGN §4.4): the band kernel's
Mehrotra predictor-corrector (scaling, start point, proximal term, step rule, stopping rule, second attempt, INFEASIBLE rule), with
the normal equations solved the way the dense kernel solves them:

  * M = A D A' dense, padded to a multiple of the tile size TS = 64 with decoupled unit rows;
  * blocked right-looking LDL' over TS x TS tiles: the diagonal tile unblocked with the band kernel's pivot rule (a non-positive pivot
    gives 1/d = 0, which decouples the row), the panel W = A21 L11^-T by row sweeps, the trailing update A22 -= W D^-1 W';
  * per Newton solve a forward substitution L t = r, t' = D^-1 t, and a backward substitution L' dy = t'.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import solve_triangular

OPTIMAL, MAXITER, NUMERR, INFEASIBLE = 0, 1, 2, 3
TS = 64


def ldl_blocked(M, ts=TS):
    """M [N, mp, mp] symmetric (mp a multiple of ts), overwritten.  Returns (L unit lower [N, mp, mp], dinv [N, mp]) with the kernel's
    pivot rule: dinv = 1/d for a positive pivot, 0 otherwise (that column of L is then 0)."""
    N, mp, _ = M.shape
    L = np.zeros_like(M)
    dinv = np.zeros((N, mp))
    for K0 in range(0, mp, ts):
        K1 = K0 + ts
        for j in range(K0, K1):                                   # diagonal tile, unblocked
            piv = M[:, j, j]
            inv = np.where(piv > 0.0, 1.0 / np.where(piv > 0.0, piv, 1.0), 0.0)
            col = M[:, j + 1:K1, j]
            M[:, j + 1:K1, j + 1:K1] -= (col * inv[:, None])[:, :, None] * col[:, None, :]
            dinv[:, j] = inv
        L11 = np.tril(M[:, K0:K1, K0:K1], -1) * dinv[:, None, K0:K1] + np.eye(ts)
        L[:, K0:K1, K0:K1] = L11
        if K1 == mp:
            break
        W = M[:, K1:, K0:K1].copy()                               # panel: W = A21 L11^-T, row sweeps
        for j in range(ts - 1):
            W[:, :, j + 1:] -= W[:, :, j:j + 1] * L11[:, None, j + 1:, j]
        Ls = W * dinv[:, None, K0:K1]
        L[:, K1:, K0:K1] = Ls
        M[:, K1:, K1:] -= Ls @ np.swapaxes(W, 1, 2)               # trailing update
    return L, dinv


def ldl_solve(L, dinv, r):
    """M v = r [N, mp] with the factor of ldl_blocked"""
    out = np.empty_like(r)
    for k in range(r.shape[0]):
        t = solve_triangular(L[k], r[k], lower=True, unit_diagonal=True, check_finite=False)
        out[k] = solve_triangular(L[k].T, dinv[k] * t, lower=False, unit_diagonal=True, check_finite=False)
    return out


def _attempt(A, b, c, u, bd, tol, feas_tol, max_iter, eta, rho, gap_floor):
    m, n = A.shape
    mp = -(-m // TS) * TS
    N = b.shape[0]
    nbnd = int(bd.sum())
    ub = np.where(bd, u, 1.0)
    x = np.ones((N, n)); x[:, bd] = np.minimum(1.0, 0.5 * ub[:, bd])
    s = np.where(bd, ub - x, 1.0)
    z = np.ones((N, n)); w_ = np.tile(np.where(bd, 1.0, 0.0), (N, 1))
    y = np.zeros((N, m))
    nb_ = 1.0 + np.abs(b).max(1); nc_ = 1.0 + (np.abs(c).max(1) > 0)
    status = np.full(N, MAXITER); iters = np.full(N, max_iter)
    active = np.ones(N, bool)
    ntot = n + nbnd
    for it in range(max_iter + 1):
        rp = b - x @ A.T
        ru = np.where(bd, ub - x - s, 0.0)
        rd = c - y @ A - z + w_
        mu = ((x * z).sum(1) + (s * w_).sum(1)) / ntot
        pobj = (c * x).sum(1); dobj = (b * y).sum(1) - (np.where(bd, ub, 0.0) * w_).sum(1)
        pres = np.maximum(np.abs(rp).max(1), np.abs(ru).max(1)) / nb_
        dres = np.abs(rd).max(1) / nc_
        gap = np.abs(pobj - dobj) / np.maximum(gap_floor, np.abs(pobj))
        res = np.maximum(pres, dres)
        cgap = ntot * mu / np.maximum(gap_floor, np.abs(pobj))
        bad = active & (~np.isfinite(mu) | ~np.isfinite(pobj) | (mu > 1e100))
        status[bad] = NUMERR; iters[bad] = it; active &= ~bad
        done = (res < feas_tol) & (gap < tol)
        done |= (cgap < tol) & (res < 10.0 * feas_tol) & (gap < 10.0 * tol)
        giveup = (cgap < 1e-3 * tol) & ~done
        done |= giveup & (res < 100.0 * feas_tol) & (gap < 1000.0 * tol)
        failed = active & giveup & ~done
        status[failed] = NUMERR; iters[failed] = it; active &= ~failed
        newly = active & done
        status[newly] = OPTIMAL; iters[newly] = it; active &= ~done
        if not active.any() or it == max_iter:
            break
        ix = np.flatnonzero(active)
        na = ix.size
        xa, sa, za, wa, ya = x[ix], s[ix], z[ix], w_[ix], y[ix]
        d = 1.0 / (za / xa + np.where(bd, wa / sa, 0.0) + rho / np.maximum(1.0, xa * xa))
        M = np.zeros((na, mp, mp))
        M[:, :m, :m] = np.einsum("ij,nj,kj->nik", A, d, A, optimize=True)
        M[:, np.arange(m, mp), np.arange(m, mp)] = 1.0            # decoupled unit rows
        L, dinv = ldl_blocked(M)

        def newton(rxz, rsw):
            h = rd[ix] - rxz / xa + np.where(bd, (rsw - wa * ru[ix]) / sa, 0.0)
            r = np.zeros((na, mp)); r[:, :m] = rp[ix] + (d * h) @ A.T
            dy = ldl_solve(L, dinv, r)[:, :m]
            dx = d * (dy @ A - h)
            ds = np.where(bd, ru[ix] - dx, 0.0)
            dz = (rxz - za * dx) / xa
            dw = np.where(bd, (rsw - wa * ds) / sa, 0.0)
            return dx, ds, dy, dz, dw

        def maxstep(v, dv, mask=None):
            r = np.where(dv < 0, -v / np.where(dv < 0, dv, -1.0), np.inf)
            if mask is not None:
                r = np.where(mask, r, np.inf)
            return r.min(1)

        dx, ds, dy, dz, dw = newton(-xa * za, -sa * wa)
        ap = np.minimum(1.0, np.minimum(maxstep(xa, dx), maxstep(sa, ds, bd)))
        ad = np.minimum(1.0, np.minimum(maxstep(za, dz), maxstep(wa, dw, bd)))
        mu_a = (((xa + ap[:, None] * dx) * (za + ad[:, None] * dz)).sum(1)
                + ((sa + ap[:, None] * ds) * (wa + ad[:, None] * dw)).sum(1)) / ntot
        sm = ((mu_a / mu[ix]) ** 3 * mu[ix])[:, None]
        dx, ds, dy, dz, dw = newton(sm - xa * za - dx * dz, np.where(bd, sm - sa * wa - ds * dw, 0.0))
        ap = np.minimum(1.0, eta * np.minimum(maxstep(xa, dx), maxstep(sa, ds, bd)))
        ad = np.minimum(1.0, eta * np.minimum(maxstep(za, dz), maxstep(wa, dw, bd)))
        x[ix] = xa + ap[:, None] * dx; s[ix] = np.where(bd, sa + ap[:, None] * ds, 1.0)
        y[ix] = ya + ad[:, None] * dy; z[ix] = za + ad[:, None] * dz; w_[ix] = np.where(bd, wa + ad[:, None] * dw, 0.0)
    return x, y, status, iters


def solve_batch(A, b, c, u, tol=1e-9, feas_tol=1e-9, max_iter=60, eta=0.9995, rho=1e-8, gap_floor=1e-4):
    """A: [m, n] (any row order, any bandwidth); b [N, m], c [N, n], u [N, n] (inf = none).  Returns dict(obj, x, y, status, iters)
    like the kernel: a bound below -1e-9 beta_b is INFEASIBLE (NaN objective and rows, iters 0); an LP whose first attempt ends
    non-optimal gets a second one (step 0.99, 10x proximal term) and reports the iterations of both."""
    A = np.asarray(A.todense() if hasattr(A, "todense") else A, float)
    m, n = A.shape
    b = np.atleast_2d(b).astype(float); c = np.atleast_2d(c).astype(float); u = np.atleast_2d(u).astype(float)
    N = b.shape[0]
    bd = np.isfinite(u[0])
    bmax = np.maximum(np.abs(b).max(1), np.where(bd, u, -np.inf).max(1, initial=-np.inf))
    beta_b = np.where(bmax > 0, bmax, 1.0)
    cmax = np.abs(c).max(1); beta_c = np.where(cmax > 0, cmax, 1.0)
    infeas = np.any(bd & (u < -1e-9 * beta_b[:, None]), axis=1)
    bs = b / beta_b[:, None]; us = np.where(bd, np.maximum(u / beta_b[:, None], 1e-10), np.inf); cs = c / beta_c[:, None]
    out = dict(obj=np.full(N, np.nan), x=np.full((N, n), np.nan), y=np.full((N, m), np.nan), status=np.full(N, INFEASIBLE),
               iters=np.zeros(N, int))
    ok = np.flatnonzero(~infeas)
    if ok.size:
        x, y, st, its = _attempt(A, bs[ok], cs[ok], us[ok], bd, tol, feas_tol, max_iter, eta, rho, gap_floor)
        redo = np.flatnonzero(st != OPTIMAL)
        if redo.size:
            x2, y2, st2, its2 = _attempt(A, bs[ok][redo], cs[ok][redo], us[ok][redo], bd, tol, feas_tol, max_iter, 0.99, 10.0 * rho, gap_floor)
            x[redo], y[redo], st[redo], its[redo] = x2, y2, st2, its[redo] + its2
        out["obj"][ok] = (cs[ok] * x).sum(1) * beta_b[ok] * beta_c[ok]
        out["x"][ok] = x * beta_b[ok, None]; out["y"][ok] = y * beta_c[ok, None]
        out["status"][ok] = st; out["iters"][ok] = its
    return out
