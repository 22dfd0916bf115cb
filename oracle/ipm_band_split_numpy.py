"""CPU ORACLE (test infrastructure -- NOT product code).

Numpy mirror of the split band kernel (dispatches_b200/csrc/dsp_band_split.cuh, DSP_KERNEL_BAND_SPLIT):

* ``split_factor`` / ``split_solve``: the scalar LDL' of P M P' for the kernel's nested-dissection permutation P of a band matrix M
  (half bandwidth W, m >= 64 W): rows cut into 32 chunks, the last W rows of chunks 0..30 separators; every interior first (the 32
  lanes in step, each on its own chunk), then the separator chain S_0..S_14, S_30..S_16, S_15.  The arrays have the kernel's
  workspace layout -- band ``Mb[k, s, L]`` (M[i][i-k] for row i = slot s of lane L), spike ``G[k, s, L]`` -- and every update is the
  kernel's expression, so the emulated kernel agrees to rounding.
* ``solve``: the band kernel's IPM (solve_one in dsp_lp.cu: scaling, start point, proximal term, stopping rule, the second attempt
  with a 100x proximal term) on one LP of an ``LPTemplate``, its normal equations solved by the two functions above.
"""
from __future__ import annotations

import numpy as np

OPTIMAL, MAX_ITER, NUMERICAL, INFEASIBLE = 0, 1, 2, 3
GAP_FLOOR = 1e-4


def layout(m):
    """rows per lane, first template row of every lane, slots per lane"""
    base, rem = divmod(m, 32)
    cs = np.array([base + (L < rem) for L in range(32)])
    r0 = np.concatenate([[0], np.cumsum(cs)])[:32]
    return cs, r0, int(cs.max())


def pack(M, W):
    """band of the dense symmetric M in split layout: Mb[k, s, L] = M[i, i-k] (0 for i-k < 0)"""
    m = M.shape[0]
    cs, r0, Sr = layout(m)
    Mb = np.zeros((W + 1, Sr, 32))
    for L in range(32):
        for s in range(cs[L]):
            i = r0[L] + s
            for k in range(min(W, i) + 1):
                Mb[k, s, L] = M[i, i - k]
    return Mb


def split_index(m):
    """v_split.flat[s * 32 + L] = v[r0[L] + s]: (split positions of the template rows, validity mask of the split slots)"""
    cs, r0, Sr = layout(m)
    pos = np.concatenate([np.arange(cs[L]) * 32 + L for L in range(32)])
    valid = np.zeros(Sr * 32, bool)
    valid[pos] = True
    return pos, valid


def _inv(d):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(d > 0.0, 1.0 / np.where(d > 0.0, d, 1.0), 0.0)


class Factor:
    def __init__(self, Mb, G, W, m):
        self.Mb, self.G, self.W, self.m = Mb, G, W, m
        self.cs, self.r0, self.Sr = layout(m)

    # separator block k: D[a, b] = M[S_k a][S_k b] (a >= b) in the band of S_k's rows, C[a, b] = M[S_k a][S_{k-1} b] in their spike
    def get_D(self, k):
        W, base = self.W, self.cs[k] - self.W
        D = np.zeros((W, W))
        for a in range(W):
            for b in range(a + 1):
                D[a, b] = self.Mb[a - b, base + a, k]
        return D

    def set_D(self, k, D):
        W, base = self.W, self.cs[k] - self.W
        for a in range(W):
            for b in range(a + 1):
                self.Mb[a - b, base + a, k] = D[a, b]

    def get_C(self, k):
        base = self.cs[k] - self.W
        return self.G[:, base:base + self.W, k].T.copy()

    def set_C(self, k, C):
        base = self.cs[k] - self.W
        self.G[:, base:base + self.W, k] = C.T


def split_factor(Mb, W, m):
    """the kernel's split_factor on a copy of the packed band; returns the Factor (band slot 0 = 1/d, other entries L * d)"""
    if m < 64 * W:
        raise ValueError("the split factorisation needs m >= 64 W")
    Mb = np.array(Mb, float)
    cs, r0, Sr = layout(m)
    lanes = np.arange(32)
    ni = np.where(lanes < 31, cs - W, cs)
    G = np.zeros((W, Sr, 32))
    for s in range(W):
        for k in range(s, W):
            G[k, s, 1:] = Mb[s + W - k, s, 1:]
    E = np.zeros((W, W, 32))
    for j in range(int(ni.max())):
        act = j < ni
        inv = _inv(Mb[0, j])
        l = [np.where((j + r < cs), Mb[r, j + r], 0.0) if j + r < Sr else np.zeros(32) for r in range(1, W + 1)]
        gj = G[:, j].copy()
        for r in range(1, W + 1):
            if j + r >= Sr:
                break
            ok = act & (j + r < cs)
            lr = l[r - 1]
            for q in range(1, r + 1):
                Mb[r - q, j + r] = np.where(ok, Mb[r - q, j + r] - lr * l[q - 1] * inv, Mb[r - q, j + r])
            G[:, j + r] = np.where(ok, G[:, j + r] - lr * gj * inv, G[:, j + r])
        for a in range(W):
            for b in range(a + 1):
                E[a, b] = np.where(act, E[a, b] - gj[a] * gj[b] * inv, E[a, b])
        Mb[0, j] = np.where(act, inv, Mb[0, j])
    F = Factor(Mb, G, W, m)
    D = [F.get_D(k) for k in range(31)]
    C = [F.get_C(k) for k in range(31)]
    low = np.tril(np.ones((W, W), bool))
    for k in range(31):
        D[k] = np.where(low, D[k] + E[:, :, k + 1], D[k])
    X = np.zeros((W, W))
    for t in range(15):
        f, h = t, 30 - t
        for p in range(W):
            invf, invh = _inv(D[f][p, p]), _inv(D[h][p, p])
            upd = low & (np.arange(W)[None, :] > p)
            colf = D[f][:, p].copy()
            D[f] = np.where(upd, D[f] - np.outer(colf, colf) * invf, D[f])
            cp = C[f + 1][:, p].copy()
            C[f + 1] = np.where(np.arange(W)[None, :] > p, C[f + 1] - np.outer(cp, colf) * invf, C[f + 1])
            D[f + 1] = np.where(low, D[f + 1] - np.outer(cp, cp) * invf, D[f + 1])
            colh = D[h][:, p].copy()
            rowh = C[h][p, :].copy()
            D[h] = np.where(upd, D[h] - np.outer(colh, colh) * invh, D[h])
            C[h] = np.where(np.arange(W)[:, None] > p, C[h] - np.outer(colh, rowh) * invh, C[h])
            if h == 16:
                X = np.where(low, X - np.outer(rowh, rowh) * invh, X)
            else:
                D[h - 1] = np.where(low, D[h - 1] - np.outer(rowh, rowh) * invh, D[h - 1])
            D[f][p, p] = invf
            D[h][p, p] = invh
    D[15] = np.where(low, D[15] + X, D[15])
    for p in range(W):
        invm = _inv(D[15][p, p])
        upd = low & (np.arange(W)[None, :] > p)
        col = D[15][:, p].copy()
        D[15] = np.where(upd, D[15] - np.outer(col, col) * invm, D[15])
        D[15][p, p] = invm
    for k in range(31):
        F.set_D(k, D[k])
        F.set_C(k, C[k])
    return F


def split_solve(F: Factor, v):
    """the kernel's split_solve: v [Sr, 32] (split layout) -> the solution of M x = v, same layout"""
    W, Mb, G, cs = F.W, F.Mb, F.G, F.cs
    Sr = F.Sr
    v = np.array(v, float)
    lanes = np.arange(32)
    ni = np.where(lanes < 31, cs - W, cs)
    D = [F.get_D(k) for k in range(31)]
    C = [F.get_C(k) for k in range(31)]
    dinv = [np.diag(D[k]).copy() for k in range(31)]
    acc = np.zeros((W, 32))
    for j in range(int(ni.max())):
        act = j < ni
        t = v[j] * Mb[0, j]
        for r in range(1, W + 1):
            if j + r >= Sr:
                break
            ok = act & (j + r < cs)
            v[j + r] = np.where(ok, v[j + r] - Mb[r, j + r] * t, v[j + r])
        acc = np.where(act & (lanes > 0), acc - G[:, j] * t, acc)
    vs = [v[cs[k] - W:cs[k], k].copy() for k in range(31)]
    for k in range(31):
        vs[k] = vs[k] + acc[:, k + 1]
    xv = np.zeros(W)
    for t in range(15):
        f, h = t, 30 - t
        for p in range(W):
            tf = vs[f][p] * dinv[f][p]
            th = vs[h][p] * dinv[h][p]
            a = np.arange(W) > p
            vs[f] = np.where(a, vs[f] - D[f][:, p] * tf, vs[f])
            vs[f + 1] = vs[f + 1] - C[f + 1][:, p] * tf
            vs[h] = np.where(a, vs[h] - D[h][:, p] * th, vs[h])
            if h == 16:
                xv = xv - C[h][p, :] * th
            else:
                vs[h - 1] = vs[h - 1] - C[h][p, :] * th
    vs[15] = vs[15] + xv
    for p in range(W):
        tm = vs[15][p] * dinv[15][p]
        vs[15] = np.where(np.arange(W) > p, vs[15] - D[15][:, p] * tm, vs[15])
    for k in range(31):
        v[cs[k] - W:cs[k], k] = vs[k]
    valid = np.arange(Sr)[:, None] < cs[None, :]
    v = np.where(valid, v * Mb[0], v)
    vs = [v[cs[k] - W:cs[k], k].copy() for k in range(31)]
    for a in range(W - 1, 0, -1):
        vs[15][:a] = vs[15][:a] - dinv[15][:a] * D[15][a, :a] * vs[15][a]
    for j in range(1, 16):
        f, h = 15 - j, 15 + j
        s = np.zeros(W)
        for a in range(W):
            s = s + C[f + 1][a, :] * vs[f + 1][a]
        vs[f] = vs[f] - dinv[f] * s
        s = np.zeros(W)
        for b in range(W):
            s = s + C[h][:, b] * vs[h - 1][b]
        vs[h] = vs[h] - dinv[h] * s
        for a in range(W - 1, 0, -1):
            vs[f][:a] = vs[f][:a] - dinv[f][:a] * D[f][a, :a] * vs[f][a]
            vs[h][:a] = vs[h][:a] - dinv[h][:a] * D[h][a, :a] * vs[h][a]
    for k in range(31):
        v[cs[k] - W:cs[k], k] = vs[k]
    sp = np.zeros((W, 32))
    for L in range(1, 32):
        sp[:, L] = v[cs[L - 1] - W:cs[L - 1], L - 1]
    for j in range(int(ni.max()) - 1, -1, -1):
        act = j < ni
        s = np.zeros(32)
        for r in range(1, W + 1):
            if j + r >= Sr:
                break
            s = np.where(j + r < cs, s + Mb[r, j + r] * v[j + r], s)
        sg = s
        for k in range(W):
            sg = sg + G[k, j] * sp[k]
        s = np.where(lanes > 0, sg, s)
        v[j] = np.where(act, v[j] - Mb[0, j] * s, v[j])
    return v


def band_solve(M, rhs, W):
    """M x = rhs for a dense symmetric band matrix M (template row order) through the split factorisation"""
    m = M.shape[0]
    pos, valid = split_index(m)
    F = split_factor(pack(M, W), W, m)
    v = np.zeros(F.Sr * 32)
    v[pos] = rhs
    return split_solve(F, v.reshape(F.Sr, 32)).reshape(-1)[pos]


# ----------------------------------------------------------------------------------------------------------------------------------
def _half_bandwidth(w):
    W = 1
    while W < w:
        W *= 2
    return W


def _band_of(A, d, m, W):
    """lower band of A diag(d) A' in split layout"""
    M = (A @ (A.T.multiply(d[:, None]))).tocsr() if hasattr(A, "tocsr") else A @ (d[:, None] * A.T)
    M = M.toarray() if hasattr(M, "toarray") else M
    return pack(M, W)


def _attempt(A, At, c, b, u, bnd, W, step_frac, reg, tol, feas_tol, max_iter):
    m, n = A.shape
    nb = int(bnd.sum())
    cs, r0, Sr = layout(m)
    pos, _ = split_index(m)
    beta_b = max(np.abs(b).max(initial=0.0), u[bnd].max(initial=0.0))
    beta_b = beta_b if beta_b > 0 else 1.0
    cmax = np.abs(c).max(initial=0.0)
    beta_c = cmax if cmax > 0 else 1.0
    if np.any(u[bnd] < -1e-9 * beta_b):
        return dict(status=INFEASIBLE, it=0, pobj=np.nan, x=None, y=None, beta_b=beta_b, beta_c=beta_c)
    b = b / beta_b
    c = c / beta_c
    uu = np.where(bnd, np.maximum(u / beta_b, 1e-10), 1.0)
    x = np.where(bnd, np.minimum(1.0, 0.5 * uu), 1.0)
    s = np.where(bnd, uu - x, 0.0)
    wv = np.where(bnd, 1.0, 0.0)
    z = np.ones(n)
    y = np.zeros(m)
    nrm_b = 1.0 + np.abs(b).max(initial=0.0)
    nrm_c = 1.0 + (1.0 if cmax > 0 else 0.0)
    ntot = float(n + nb)
    status, pobj = MAX_ITER, 0.0
    it = 0
    for it in range(max_iter + 1):
        rp = b - A @ x
        rd = c - z - At @ y + wv
        rx = 1.0 / x
        t = z * rx + np.where(x > 1.0, reg * rx * rx, reg)
        ru = np.where(bnd, uu - x - s, 0.0)
        rs = np.where(bnd, 1.0 / np.where(bnd, s, 1.0), 0.0)
        t = t + wv * rs
        d = 1.0 / t
        pmax = max(np.abs(rp).max(initial=0.0), np.abs(ru).max(initial=0.0))
        dmax = np.abs(rd).max(initial=0.0)
        mu = ((x * z).sum() + (s * wv).sum()) / ntot
        po = float(c @ x)
        dobj = float(b @ y) - float((uu * wv)[bnd].sum())
        pobj = po
        gap = abs(po - dobj) / max(GAP_FLOOR, abs(po))
        if not np.isfinite(mu) or not np.isfinite(po) or mu > 1e100:
            status = NUMERICAL
            break
        res = max(pmax / nrm_b, dmax / nrm_c)
        cgap = ntot * mu / max(GAP_FLOOR, abs(po))
        if res < feas_tol and gap < tol:
            status = OPTIMAL
            break
        if cgap < tol and res < 10.0 * feas_tol and gap < 10.0 * tol:
            status = OPTIMAL
            break
        if cgap < 1e-3 * tol:
            status = OPTIMAL if (res < 100.0 * feas_tol and gap < 1000.0 * tol) else NUMERICAL
            break
        if it == max_iter:
            break
        F = split_factor(_band_of(A, d, m, W), W, m)

        def newton(corr, smu):
            h = rd + z
            if corr is not None:
                cor, cors = corr
                h = h - (smu - cor) * rx
            as_ = -wv * ru + (smu - cors if corr is not None else 0.0)
            h = np.where(bnd, h + as_ * rs - wv, h)
            dx0 = d * h
            v = np.zeros(Sr * 32)
            v[pos] = rp + A @ dx0
            dy = split_solve(F, v.reshape(Sr, 32)).reshape(-1)[pos]
            return d * (At @ dy) - dx0, dy

        def steps(dx, corr, smu):
            dz = -z - z * dx * rx
            ds = ru - dx
            dw = -wv - wv * ds * rs
            if corr is not None:
                dz = dz + (smu - corr[0]) * rx
                dw = dw + (smu - corr[1]) * rs
            ip = max(0.0, (-dx * rx).max(initial=0.0), np.where(bnd, -ds * rs, 0.0).max(initial=0.0))
            idd = max(0.0, (-dz / z).max(initial=0.0), np.where(bnd, -dw / np.where(bnd, wv, 1.0), 0.0).max(initial=0.0))
            return ip, idd, dz, ds, dw

        dx, dy = newton(None, 0.0)
        ip, idd, dz, ds, dw = steps(dx, None, 0.0)
        ap = 1.0 / ip if ip > 1.0 else 1.0
        ad = 1.0 / idd if idd > 1.0 else 1.0
        mua = (((x + ap * dx) * (z + ad * dz)).sum() + np.where(bnd, (s + ap * ds) * (wv + ad * dw), 0.0).sum()) / ntot
        cor = dx * dz
        cors = np.where(bnd, ds * dw, 0.0)
        sg = mua / mu
        smu = sg * sg * sg * mu
        dx, dy = newton((cor, cors), smu)
        ip, idd, dz, ds, dw = steps(dx, (cor, cors), smu)
        ap = step_frac / ip if step_frac < ip else 1.0
        ad = step_frac / idd if step_frac < idd else 1.0
        s = np.where(bnd, s + ap * ds, s)
        wv = np.where(bnd, wv + ad * dw, wv)
        x = x + ap * dx
        z = z + ad * dz
        y = y + ad * dy
    return dict(status=status, it=it, pobj=pobj, x=x * beta_b, y=y * beta_c, beta_b=beta_b, beta_c=beta_c)


def solve(t, cparams, rparams, tol=1e-9, feas_tol=1e-9, max_iter=60, step_frac=0.9995, reg=1e-8):
    """one LP of the LPTemplate t (finalized: band row order, bounded columns first) as DSP_KERNEL_BAND_SPLIT solves it, without the
    band kernel's retry: dict(obj, status, iters, x, y)"""
    c, b, u, k = t.instantiate(cparams, rparams)
    A = t.A.tocsr()
    At = A.T.tocsr()
    bnd = np.isfinite(t.u0)
    u = np.where(bnd, u, 0.0)
    W = _half_bandwidth(t.w)
    r = _attempt(A, At, c, b, u, bnd, W, step_frac, reg, tol, feas_tol, max_iter)
    it0 = r["it"]
    if r["status"] == INFEASIBLE:
        return dict(obj=np.nan, status=INFEASIBLE, iters=0, x=None, y=None)
    if r["status"] != OPTIMAL:
        r = _attempt(A, At, c, b, u, bnd, W, 0.99, 100.0 * reg, tol, feas_tol, max_iter)
        r["it"] += it0
    return dict(obj=r["pobj"] * r["beta_b"] * r["beta_c"] + k, status=r["status"], iters=r["it"], x=r["x"], y=r["y"])
