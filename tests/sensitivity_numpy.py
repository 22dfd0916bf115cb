"""numpy mirror of the sensitivity post-pass (include/dsp_lp.h: dsp_lp_sensitivities, csrc/dsp_sens.cuh).

For one LP  min c'x + k  s.t.  A x = b, 0 <= x <= u  of an LPTemplate at (cparams, rparams) with a returned (x, y):

    rc            = c - A'y                     A = t.matrix(rparams): A0 plus the per-problem matrix terms
    d obj / d cp  = Cmap' x + ocmap
    d obj / d rp  = Bmap' y + Umap' min(rc, 0) + omap - sum over the matrix terms (i, j, q, coef) of coef * y_i * x_j

the convention of tests/exact_lp.py::kkt_residuals (min(rc, 0) = -w, the upper-bound dual that is optimal for this y).  Works in
template order, the order BatchLPSolver returns x and y in.  ``scales`` returns, per entry, the sum of the absolute values of its terms:
the scale a rounding error of the entry is measured against (an entry that cancels to ~0 has no relative accuracy of its own).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def _rows(a, N):
    a = np.asarray(a, float)
    return np.broadcast_to(a, (N, a.shape[-1])) if a.ndim == 1 else a


def sensitivities(t, cparams, rparams, x, y, status=None):
    """(rc [N,n], d_cparams [N,Pc], d_rparams [N,Pr]); rows of NaN where status != 0"""
    x = np.atleast_2d(np.asarray(x, float)); y = np.atleast_2d(np.asarray(y, float))
    N = x.shape[0]
    cp = _rows(np.zeros((N, 0)) if t.Pc == 0 else cparams, N)
    rp = _rows(np.zeros((N, 0)) if t.Pr == 0 else rparams, N)
    Cm, Bm, Um = t.Cmap.tocsr(), t.Bmap.tocsr(), t.Umap.tocsr()
    fin = np.isfinite(t.u0)
    rc = np.empty((N, t.n)); dcp = np.empty((N, t.Pc)); drp = np.empty((N, t.Pr))
    for k in range(N):
        c, _, _, _ = t.instantiate(cp[k], rp[k])
        A = t.matrix(rp[k]).tocsr()
        r = c - A.T @ y[k]
        rc[k] = r
        dcp[k] = Cm.T @ x[k] + t.ocmap
        d = Bm.T @ y[k] + Um.T @ np.where(fin, np.minimum(r, 0.0), 0.0) + t.omap
        if t.amap is not None:
            for i, j, q, v in zip(*t.amap):
                d[q] -= v * y[k, i] * x[k, j]
        drp[k] = d
    if status is not None:
        bad = np.asarray(status) != 0
        rc[bad] = np.nan; dcp[bad] = np.nan; drp[bad] = np.nan
    return rc, dcp, drp


def scales(t, cparams, rparams, x, y):
    """per entry of (rc, d_cparams, d_rparams): the sum of the absolute values of its terms"""
    x = np.atleast_2d(np.asarray(x, float)); y = np.atleast_2d(np.asarray(y, float))
    N = x.shape[0]
    cp = _rows(np.zeros((N, 0)) if t.Pc == 0 else cparams, N)
    rp = _rows(np.zeros((N, 0)) if t.Pr == 0 else rparams, N)
    Cm, Bm, Um = abs(t.Cmap.tocsr()), abs(t.Bmap.tocsr()), abs(t.Umap.tocsr())
    fin = np.isfinite(t.u0)
    src = np.empty((N, t.n)); sdc = np.empty((N, t.Pc)); sdr = np.empty((N, t.Pr))
    for k in range(N):
        A = abs(t.A.tocsr())                  # |A0| plus |coef rp[param]| of every matrix term: the terms an entry of A sums
        if t.amap is not None:
            i, j, q, v = t.amap
            A = A + sp.csr_matrix((np.abs(v * rp[k][q]), (i, j)), shape=A.shape)
        s = np.abs(t.c0) + Cm @ np.abs(cp[k]) + A.T @ np.abs(y[k])
        src[k] = s
        sdc[k] = Cm.T @ np.abs(x[k]) + np.abs(t.ocmap)
        d = Bm.T @ np.abs(y[k]) + Um.T @ np.where(fin, s, 0.0) + np.abs(t.omap)
        if t.amap is not None:
            for i, j, q, v in zip(*t.amap):
                d[q] += abs(v * y[k, i] * x[k, j])
        sdr[k] = d
    return src, sdc, sdr


def rel_err(a, b, scale):
    """max |a - b| / max(scale, tiny), NaN where both are NaN counting as equal"""
    a = np.asarray(a, float); b = np.asarray(b, float)
    both = np.isnan(a) & np.isnan(b)
    if np.any(np.isnan(a) != np.isnan(b)):
        return np.inf
    d = np.where(both, 0.0, np.abs(a - b)) / np.maximum(np.where(both, 1.0, scale), 1e-300)
    return float(d.max()) if d.size else 0.0
