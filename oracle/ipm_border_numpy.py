"""CPU ORACLE (test infrastructure -- NOT product code).

Batched numpy mirror of the band kernel with LINKING COLUMNS (dispatches_b200/csrc/dsp_lp.cu, DESIGN §4.3): the same Mehrotra
predictor-corrector as oracle/ipm_numpy.py (scaling, start point, proximal term, step rule, stopping rule, second attempt), but the
normal equations are solved the way the kernel solves them when the template has a border ``A = [A_s | A_b]``:

  1. the band of  M_s = A_s D_s A_s'  (rows in template order, half bandwidth w), factorised by band LDL' in row order with a
     PIVOT GUARD: a pivot p below  EPS * GAMMA,  GAMMA = the largest diagonal of M_s, is replaced by GAMMA and its row recorded with
     the shift  delta = GAMMA - p  (Andersen's modified Schur complement, ACM TOMS 22(3), 1996).  The factor is that of
     M~ = M_s + sum delta_i e_i e_i',  and  M = M~ + V E V'  with  V = [A_b, e_i ...],  E = diag(D_b, -delta ...).  The threshold is
     relative to GAMMA, not to the row's own diagonal: the rows a basic linking column carries have tiny diagonals of their own
     (their sparse columns are nonbasic), so a test against the row's diagonal does not see them go singular;
  2. Z = M~^-1 V  (k + q right-hand sides) and  S = E^-1 + V'Z  (small, indefinite: LU with partial pivoting);
  3. every Newton solve:  v = M~^-1 r,  t = S^-1 V'v,  dy = v - Z t.

A plain Schur complement on M_s^-1 fails once a border column is basic (M_s is then singular up to the proximal term: DESIGN §6b);
the guard turns those near-zero pivots into rank-one corrections that the small system absorbs.
"""
from __future__ import annotations

import numpy as np

OPTIMAL, MAXITER, NUMERR, INFEASIBLE = 0, 1, 2, 3
EPS = 1e-12          # guard threshold relative to the largest diagonal of M_s
REFINE = 0           # steps of iterative refinement on the true M per Newton solve
KMAX = 8             # linking columns; the guarded rows are capped at the same number


def _band_factor_guarded(Mb, w, kcap, eps=EPS):
    """Mb [N, m + w, w + 1] (w zero rows behind), Mb[:, i, k] = M[i, i-k].  In place: the diagonal slot gets 1/pivot, the off-diagonal
    slots the unscaled L entries (the kernel's storage).  A pivot p <= EPS * gamma (gamma = the largest diagonal of M_s) becomes gamma:
    the factor is then that of M_s + (gamma - p) e_i e_i'.  Returns (guarded rows [N, kcap] (-1 = none), their shifts gamma - p [N, kcap],
    count [N], gamma [N])."""
    N, mp, _ = Mb.shape
    m = mp - w
    diag0 = Mb[:, :m, 0].copy()
    gamma = np.maximum(diag0.max(1), 1e-300)
    rr, qq = np.meshgrid(np.arange(1, w + 1), np.arange(1, w + 1), indexing="ij")
    sel = qq <= rr
    rr, qq = rr[sel], qq[sel]
    guard = -np.ones((N, kcap), int)
    shift = np.zeros((N, kcap))
    cnt = np.zeros(N, int)
    ar = np.arange(N)
    for j in range(m):
        piv = Mb[:, j, 0]
        bad = ~(piv > eps * gamma)
        if bad.any():
            ok = bad & (cnt < kcap)
            guard[ar[ok], cnt[ok]] = j
            shift[ar[ok], cnt[ok]] = gamma[ok] - piv[ok]
            piv = np.where(bad, gamma, piv)
            cnt = cnt + bad
        inv = 1.0 / piv
        L = Mb[:, j + np.arange(1, w + 1), np.arange(1, w + 1)] if w else np.zeros((N, 0))
        if w:
            Mb[:, j + rr, rr - qq] -= L[:, rr - 1] * L[:, qq - 1] * inv[:, None]
        Mb[:, j, 0] = inv
    return guard, shift, cnt, gamma


def _band_solve(Mb, v, w):
    """v [N, m + w, R] in place (w zero entries behind): M~ v = r with the factor of _band_factor_guarded."""
    N, mp, _ = Mb.shape
    m = mp - w
    rng = np.arange(1, w + 1)
    for j in range(m):
        t = v[:, j] * Mb[:, j, 0][:, None]
        if w:
            v[:, j + rng] -= Mb[:, j + rng, rng][:, :, None] * t[:, None, :]
    v[:, :m] *= Mb[:, :m, 0][:, :, None]
    for i in range(m - 1, 0, -1):
        r = rng[rng <= i]
        v[:, i - r] -= (Mb[:, i - r, 0] * Mb[:, i, r])[:, :, None] * v[:, i][:, None, :]
    return v


def _small_solve(S, r):
    """S [N, R, R] t = r [N, R] by LU with partial pivoting; an exactly singular S gives NaN (the LP then ends NUMERICAL)"""
    try:
        return np.linalg.solve(S, r[:, :, None])[:, :, 0]
    except np.linalg.LinAlgError:
        out = np.full(r.shape, np.nan)
        for i in range(S.shape[0]):
            try:
                out[i] = np.linalg.solve(S[i], r[i])
            except np.linalg.LinAlgError:
                pass
        return out


def _attempt(A, border, w, b, c, u, bd, tol, feas_tol, max_iter, eta, rho, gap_floor, eps, refine):
    m, n = A.shape
    N = b.shape[0]
    Ab = A[:, border]
    k = border.size
    kc = k                                  # guarded rows: at most as many as linking columns
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
    As = A.copy(); As[:, border] = 0.0
    # band assembly pattern: M_s[i, i-kk] = sum_j As[i, j] As[i-kk, j] d_j
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
        # band of M_s
        Mb = np.zeros((na, m + w, w + 1))
        for kk in range(w + 1):
            Mb[:, kk:m, kk] = np.einsum("ij,nj,ij->ni", As[kk:], d, As[:m - kk], optimize=True)
        guard, shift, cnt, gamma = _band_factor_guarded(Mb, w, kc, eps)
        over = cnt > kc
        q = min(int(cnt.max()), kc)
        R = k + q
        V = np.zeros((na, m + w, R))
        V[:, :m, :k] = Ab[None]
        Einv = np.zeros((na, R))
        Einv[:, :k] = 1.0 / d[:, border]
        for g in range(q):
            has = guard[:, g] >= 0
            V[np.flatnonzero(has), guard[has, g], k + g] = 1.0
            Einv[:, k + g] = np.where(has, -1.0 / np.where(has, shift[:, g], 1.0), 1.0)   # unused slot: identity row / column of S
        Z = _band_solve(Mb, V.copy(), w)
        S = np.einsum("nir,nis->nrs", V[:, :m], Z[:, :m])
        S[:, np.arange(R), np.arange(R)] += Einv
        for g in range(q):                                         # unused slots: no coupling
            has = guard[:, g] >= 0
            S[~has, k + g, :] = 0.0; S[~has, :, k + g] = 0.0; S[~has, k + g, k + g] = 1.0

        def msolve0(rhs):
            v = np.zeros((na, m + w, 1)); v[:, :m, 0] = rhs
            v = _band_solve(Mb, v, w)
            t = _small_solve(S, np.einsum("nir,ni->nr", V[:, :m], v[:, :m, 0]))
            return v[:, :m, 0] - np.einsum("nir,nr->ni", Z[:, :m], t)

        def msolve(rhs):
            dy = msolve0(rhs)
            for _ in range(refine):                                # iterative refinement on the true M = A D A'
                dy = dy + msolve0(rhs - (d * (dy @ A)) @ A.T)
            return dy

        def newton(rxz, rsw):
            h = rd[ix] - rxz / xa + np.where(bd, (rsw - wa * ru[ix]) / sa, 0.0)
            dy = msolve(rp[ix] + (d * h) @ A.T)
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
        if over.any():                                             # more guarded pivots than linking columns
            status[ix[over]] = NUMERR; iters[ix[over]] = it; active[ix[over]] = False
    return x, y, z, w_, status, iters



def solve_batch(A, b, c, u, border, w, tol=1e-9, feas_tol=1e-9, max_iter=60, eta=0.9995, rho=1e-8, gap_floor=1e-4, eps=EPS, refine=REFINE):
    """A: [m, n] (template row order: M_s is banded with half bandwidth w once the ``border`` columns are left out);
    b [N, m], c [N, n], u [N, n] (inf = none).  Returns dict(obj, x, y, status, iters) like the kernel: a negative bound is
    INFEASIBLE (NaN objective, iters 0); an LP whose first attempt ends non-optimal gets a second one (step 0.99, 10x proximal
    term) and reports the iterations of both."""
    A = np.asarray(A.todense() if hasattr(A, "todense") else A, float)
    border = np.asarray(border, int)
    if border.size > KMAX:
        raise ValueError(f"at most {KMAX} linking columns")
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
        x, y, z, ww, st, its = _attempt(A, border, w, bs[ok], cs[ok], us[ok], bd, tol, feas_tol, max_iter, eta, rho, gap_floor, eps, refine)
        redo = np.flatnonzero(st != OPTIMAL)
        if redo.size:
            x2, y2, z2, w2, st2, its2 = _attempt(A, border, w, bs[ok][redo], cs[ok][redo], us[ok][redo], bd, tol, feas_tol, max_iter, 0.99,
                                                 10.0 * rho, gap_floor, eps, refine)
            x[redo], y[redo], st[redo], its[redo] = x2, y2, st2, its[redo] + its2
        out["obj"][ok] = (cs[ok] * x).sum(1) * beta_b[ok] * beta_c[ok]
        out["x"][ok] = x * beta_b[ok, None]; out["y"][ok] = y * beta_c[ok, None]
        out["status"][ok] = st; out["iters"][ok] = its
    return out
