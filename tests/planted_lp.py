"""Planted-optimum LPs (test infrastructure, no GPU): seeded standard-form LPs

    min c'x + k   s.t.  A x = b,  0 <= x <= u

whose unique optimum (x*, y*) is known by construction, for checking the band kernel against an exact answer at any
half bandwidth, size and parameter layout.

Construction.  A is a staircase: row i owns one column with a dominant entry (|a| in [4, 8]) that also touches the next rows
with small entries, and a coupling column that touches rows i .. i + w.  Rows i and i + k then share a column iff k <= w, so
the half bandwidth of A A' is exactly w in any row order a bandwidth-reducing ordering can find (every w + 1 consecutive rows
form a clique).  The m owned columns are the basis: lower triangular with a dominant diagonal, hence well conditioned.
x_B lies strictly inside its bounds (margin >= 0.1 of the range, or >= 1 when unbounded), every nonbasic column sits at 0 or
at its upper bound, and c = A'y* + r with |r_N| in [0.1, 10] and the sign complementarity asks for.  Nondegeneracy plus strict
complementarity make x* and y* unique.

Every number is a dyadic rational with few significant bits (powers of two scale it), so b = A x*, c = A'y* + r, the
parameter maps and the objective are EXACT in binary64: the reference is the optimum of the very LP the solver receives.
The objective is summed with math.fsum.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import scipy.sparse as sp

from dispatches_b200.lp_template import INF, LPTemplate

# H100 (sm_90): opt-in shared memory per block and SM count, for band_placement() below
H100_SMEM_OPTIN = 232448
H100_SMS = 132
KMAX_WARPS = 16


def _dy(rng, lo, hi, bits, size=None):
    """dyadic rationals k / 2^bits uniformly drawn in [lo, hi]"""
    s = 2.0 ** bits
    return rng.integers(int(math.ceil(lo * s)), int(math.floor(hi * s)) + 1, size=size) / s


@dataclasses.dataclass
class PlantedLP:
    t: LPTemplate              # finalized template (caller order = the template's own order)
    cparams: np.ndarray        # [N, Pc]
    rparams: np.ndarray        # [N, Pr]
    x: np.ndarray              # [N, n] planted primal, template column order
    y: np.ndarray              # [N, m] planted row duals, template row order
    obj: np.ndarray            # [N] c'x* + k, exact (math.fsum of exact products)
    lp_mag: np.ndarray         # [N] sum_j |c_j x*_j|: the magnitude of the LP part c'x* (the objective constant k excluded)
    w: int                     # requested half bandwidth of A A'
    unique_x: bool = True      # False for all-zero c: every feasible x is optimal
    unique_y: bool = True      # False for all-zero b: x* = 0 is a degenerate vertex
    scale: float = 1.0         # largest |x*| (and u of the active bounds): the primal scale of the batch


def planted(m, w, seed=0, N=1, bounded="mixed", extra=1, full_span=False, amap=False, c_scale=1.0, b_scale=1.0,
            u_scale=1.0, zero_c=False, zero_b=False, shared_rparams=False):
    """A batch of N planted LPs over one template.

    m rows, half bandwidth w (0 <= w; w > m - 1 is capped by m), ``extra`` additional coupling columns per row (grow n, nnz and the
    band-assembly list without changing w; each spans a random 1 .. w + 1 rows, or w + 1 with ``full_span``), ``bounded`` in
    {"mixed", "none", "all"}: which columns carry a finite upper bound.
    ``amap``: per-LP matrix coefficients on the coupling columns (A[row, col] = A0 + coef * rparams[..]); each LP is planted
    against its own matrix.  ``c_scale`` / ``b_scale`` scale c (and y*) / b, u and x*; ``u_scale`` multiplies only the upper
    bounds no optimal x touches (a loose box).  ``zero_c``: c = 0, objective = k.  ``zero_b``: b = 0, x* = 0.
    ``shared_rparams``: one rparams row serves the batch (b, u and amap the same for every LP; only c varies).
    """
    rng = np.random.default_rng(seed)
    we = min(w, m - 1)
    # ---- columns: (rows, values) in caller order
    cols = []
    own = []
    for i in range(m):
        span = list(range(i, min(m, i + 1 + min(we, 2))))
        vals = [float(_dy(rng, 4, 8, 2)) * rng.choice([-1.0, 1.0])] + [float(_dy(rng, -0.5, 0.5, 3)) or 0.125 for _ in span[1:]]
        own.append(len(cols)); cols.append((span, vals))
    coupling = []
    for i in range(m):
        for e in range(extra + 1):
            wide = e == 0 or full_span
            span = list(range(i, min(m, i + 1 + (we if wide else int(rng.integers(0, we + 1))))))
            vals = [float(v) if v != 0 else 0.25 for v in _dy(rng, -1, 1, 3, len(span))]
            coupling.append(len(cols)); cols.append((span, vals))
    n = len(cols)
    # shuffle the columns so that bounded / unbounded and basic / nonbasic are interleaved in caller order
    order = rng.permutation(n)
    cols = [cols[k] for k in order]
    inv = np.empty(n, int); inv[order] = np.arange(n)
    basic = np.zeros(n, bool); basic[inv[own]] = True
    ri, ci, vv = [], [], []
    for j, (rows, vals) in enumerate(cols):
        for r, v in zip(rows, vals):
            ri.append(r); ci.append(j); vv.append(v)
    A0 = sp.csr_matrix((vv, (ri, ci)), shape=(m, n))
    A0.sort_indices()
    # ---- bounds
    if bounded == "all":
        fin = np.ones(n, bool)
    elif bounded == "none":
        fin = np.zeros(n, bool)
    else:
        fin = rng.random(n) < 0.5
    nb = int(fin.sum())
    # ---- matrix parameters: one per coupling column entry of every third row
    am = None
    Pr_b = m                                            # rparams: [b-terms (m) | u-terms (nb) | b global | amap terms]
    if amap:
        rows, colsj = [], []
        for j, (rr, _) in enumerate(cols):
            if not basic[j] and rr[0] % 3 == 0:
                rows.append(rr[-1]); colsj.append(j)
        na = len(rows)
        am = (np.array(rows, int), np.array(colsj, int), Pr_b + nb + 1 + np.arange(na), _dy(rng, 0.5, 2, 2, na))
    Pr = m + nb + 1 + (0 if am is None else len(am[0]))
    Pc = n + 1
    # ---- parameter maps (fixed per template): c = c0 + g*cp[j] + e*cp[n], b = b0 + h*rp[i] + f*rp[global], u likewise
    g = rng.choice([0.5, 1.0, 2.0], n); e = _dy(rng, -1, 1, 2, n)
    h = rng.choice([0.5, 1.0, 2.0], m); f = _dy(rng, -1, 1, 2, m)
    hu = rng.choice([0.5, 1.0, 2.0], nb); fu = _dy(rng, 0, 1, 2, nb)
    c0 = _dy(rng, -4, 4, 4, n); b0 = _dy(rng, -4, 4, 4, m); u0 = np.full(n, INF)
    fidx = np.flatnonzero(fin)
    u0[fidx] = _dy(rng, 0, 2, 4, nb)
    Cmap = sp.csr_matrix((np.concatenate([g, e]), (np.r_[np.arange(n), np.arange(n)], np.r_[np.arange(n), np.full(n, n)])),
                         shape=(n, Pc))
    Bmap = sp.csr_matrix((np.concatenate([h, f]), (np.r_[np.arange(m), np.arange(m)], np.r_[np.arange(m), np.full(m, Pr_b + nb)])),
                         shape=(m, Pr))
    Umap = sp.csr_matrix((np.concatenate([hu, fu]), (np.r_[fidx, fidx], np.r_[m + np.arange(nb), np.full(nb, Pr_b + nb)])),
                         shape=(n, Pr))
    o0 = float(_dy(rng, -8, 8, 3)); omap = _dy(rng, -1, 1, 3, Pr); ocmap = _dy(rng, -1, 1, 3, Pc)
    if zero_b:
        b0[:] = 0.0
    if zero_c:
        c0[:] = 0.0
    # ---- one planted LP per slot
    CP = np.zeros((N, Pc)); RP = np.zeros((N, Pr)); X = np.zeros((N, n)); Y = np.zeros((N, m)); OBJ = np.zeros(N); MAG = np.zeros(N)
    nshared = 1 if shared_rparams else N
    for k in range(N):
        if k < nshared:
            rglob = float(_dy(rng, -1, 1, 3))
            rp = np.zeros(Pr); rp[Pr_b + nb] = rglob
            if am is not None:
                rp[am[2]] = _dy(rng, -0.5, 0.5, 3, len(am[0]))
            Ak = A0 if am is None else _with_amap(A0, am, rp)
            # primal: x_B strictly inside, nonbasic at 0 or at u
            u = np.full(n, INF); x = np.zeros(n)
            u[fin] = _dy(rng, 2, 8, 2, nb) * b_scale
            at_u = fin & ~basic & (rng.random(n) < 0.5) & (not zero_b)
            x[at_u] = u[at_u]
            bounded_basic = basic & fin
            x[basic & ~fin] = _dy(rng, 1, 4, 6, int((basic & ~fin).sum())) * b_scale
            x[bounded_basic] = u[bounded_basic] * _dy(rng, 0.125, 0.875, 6, int(bounded_basic.sum()))
            if zero_b:
                x[:] = 0.0
            b = Ak @ x
            # loose boxes: bounds no optimal x touches (basic bounded columns, nonbasic at 0) grow by u_scale
            loose = fin & ~at_u
            u[loose] = u[loose] * u_scale
            if zero_b:
                b[:] = 0.0
            # rparams that reproduce b and u exactly through the maps
            rp[:m] = (b - b0 - f * rglob) / h
            rp[m:m + nb] = (u[fidx] - u0[fidx] - fu * rglob) / hu
        else:
            rp = RP[0]; Ak = A0 if am is None else _with_amap(A0, am, rp)
            x = X[0].copy(); b = Ak @ x
            u = np.full(n, INF); u[fidx] = u0[fidx] + hu * rp[m:m + nb] + fu * rp[Pr_b + nb]
            at_u = fin & (x == u) & ~basic
        # dual: y* random, r_B = 0, r_N > 0 at 0, < 0 at u
        if zero_c:
            y = np.zeros(m); c = np.zeros(n)
        else:
            y = _dy(rng, -2, 2, 4, m) * c_scale
            r = _dy(rng, 0.125, 10, 3, n) * c_scale
            r[at_u] = -r[at_u]
            r[basic] = 0.0
            if zero_b:
                r = np.abs(r); r[basic] = _dy(rng, 0.125, 10, 3, m) * c_scale   # x* = 0: every column strictly priced out
            c = Ak.T @ y + r
        cglob = float(_dy(rng, -1, 1, 3))
        cp = np.zeros(Pc); cp[n] = cglob
        cp[:n] = (c - c0 - e * cglob) / g
        # the maps must reproduce the planted data exactly (dyadic data: no rounding anywhere)
        assert np.array_equal(c0 + g * cp[:n] + e * cglob, c)
        assert np.array_equal(b0 + h * rp[:m] + f * rp[Pr_b + nb], b)
        CP[k], RP[k], X[k], Y[k] = cp, rp, x, y
        OBJ[k] = math.fsum(list(c * x) + [o0] + list(omap * rp) + list(ocmap * cp))
        MAG[k] = math.fsum(np.abs(c * x))
    t = LPTemplate(f"planted(m={m},w={w})", A0.copy(), b0, Bmap, c0, Cmap, u0, Umap, o0, omap, ocmap,
                   np.zeros(n), np.ones(n), [f"x{j}" for j in range(n)], [f"r{i}" for i in range(m)])
    t.amap = am
    t.finalize()
    # the planted vectors in the finalized template's order
    cpos = np.array([int(nm[1:]) for nm in t.col_names]); rpos = np.array([int(nm[1:]) for nm in t.row_names])
    scale = max(1.0, float(np.abs(X).max()))
    return PlantedLP(t, CP, RP, X[:, cpos], Y[:, rpos], OBJ, MAG, w, unique_x=not zero_c, unique_y=not (zero_c or zero_b), scale=scale)


def _with_amap(A0, am, rp):
    A = A0.tolil(copy=True)
    for i, j, kk, v in zip(*am):
        A[i, j] = A[i, j] + v * rp[kk]
    return A.tocsr()


def lp_matrix(p: PlantedLP, k):
    """the constraint matrix of LP k in the finalized template's order"""
    return p.t.matrix(p.rparams[k])


def optimality(p: PlantedLP, k):
    """KKT residuals and complementarity margins of the planted (x*, y*) of LP k.  Residuals are relative to the data's scale;
    margins are the smallest distance of a basic x to its bounds (relative to the range, or absolute when unbounded) and
    the smallest |reduced cost| of a nonbasic column."""
    c, b, u, _ = p.t.instantiate(p.cparams[k], p.rparams[k])
    A = lp_matrix(p, k)
    x, y = p.x[k], p.y[k]
    r = c - A.T @ y
    fin = np.isfinite(u)
    sb = max(1.0, np.abs(b).max(), np.abs(x).max())
    sc = max(1e-300, np.abs(c).max())
    at_lo, at_hi = x == 0.0, fin & (x == u)
    inside = ~at_lo & ~at_hi
    rng_ = np.where(fin, u, 1.0)
    return dict(
        primal=np.abs(A @ x - b).max() / sb,
        bounds=max(0.0, -x.min(), np.max((x - u)[fin], initial=0.0)) / sb,
        dual=np.abs(r[inside]).max(initial=0.0) / sc,                          # basic columns: reduced cost 0
        sign=max(np.max(-r[at_lo], initial=0.0), np.max(r[at_hi], initial=0.0)) / sc,   # at 0: r >= 0, at u: r <= 0
        x_margin=np.min(np.minimum(x, np.where(fin, u - x, np.inf))[inside] / rng_[inside], initial=np.inf),
        r_margin=np.min(np.abs(r[~inside]), initial=np.inf),
        n_basic=int(inside.sum()))


def rel(a, ref):
    """largest |a - ref| of each LP relative to that LP's |ref|_inf (absolute where ref = 0): basic columns are >= 1 and bounds >= 2
    unless a test scales the data down, so this is 1e-6 * max(1, |x*|) of the planted LPs and as tight on scaled ones"""
    s = np.abs(ref).max(1)
    return float((np.abs(a - ref).max(1) / np.where(s > 0, s, 1.0)).max(initial=0.0))


def shuffled(t: LPTemplate, seed):
    """the same LPs with rows and columns in a random caller order (for dsp_lp_template_create_csr, whose own ordering and
    xperm / yperm write-back then matter).  Returns (template, column order, row order): column j of the new template is column
    cperm[j] of t, row i is row rperm[i]."""
    rng = np.random.default_rng(seed)
    cperm = rng.permutation(t.n); rperm = rng.permutation(t.m)
    s = dataclasses.replace(t, A=t.A.tocsr()[rperm][:, cperm].tocsr(), b0=t.b0[rperm], Bmap=t.Bmap.tocsr()[rperm],
                            c0=t.c0[cperm], Cmap=t.Cmap.tocsr()[cperm], u0=t.u0[cperm], Umap=t.Umap.tocsr()[cperm],
                            col_shift=t.col_shift[cperm], col_scale=t.col_scale[cperm],
                            col_names=[t.col_names[j] for j in cperm], row_names=[t.row_names[i] for i in rperm],
                            meta=dict(t.meta))
    if t.amap is not None:
        ic = np.empty(t.n, int); ic[cperm] = np.arange(t.n)
        ir = np.empty(t.m, int); ir[rperm] = np.arange(t.m)
        s.amap = (ir[t.amap[0]], ic[t.amap[1]], t.amap[2], t.amap[3])
    return s, cperm, rperm


# ---------------------------------------------------------------------------------------------------------------------
# band-kernel test cases (tests/test_band_kernel_planted.py runs them on the GPU, tests/test_planted_lp.py checks on the CPU that
# each lands in its placement).  Placements (csrc/dsp_lp.cu, band_geometry): smem_staged -- work regions and the template in shared
# memory; smem_l2 -- work regions in shared memory, template read through L2; hybrid -- work regions in a global workspace, the
# (dy, band) tail in shared memory; ws -- everything in the workspace.
#
# Two pairs cannot occur on an H100 (227 KB of shared memory per block): (1, smem_l2) and (2, smem_l2).  The template is read
# through L2 only when staging it leaves room for fewer than 4 work regions while at least 7 fit without it -- the template blob
# must exceed ~3x a work region -- or when 4-6 fit and fewer than 6 band tails do, which needs the band tail to be over 3/4 of the
# work region.  At W = 1 (2) a column costs the blob at most 88 (148) bytes against 64 in the work region and a row 12 (16)
# against 48 (56), and the band tail is under 1/4 of the region: neither condition can hold.
# ---------------------------------------------------------------------------------------------------------------------
UNREACHABLE = {(1, "smem_l2"), (2, "smem_l2")}

# (W, placement) -> planted() shape (seed 0) that lands there
CASES = {
    (1, "smem_staged"): dict(m=1, w=0),
    (1, "hybrid"): dict(m=64, w=1, extra=2, bounded="all"),
    (1, "ws"): dict(m=1700, w=1, extra=0, bounded="none"),
    (2, "smem_staged"): dict(m=3, w=2, bounded="all"),
    (2, "hybrid"): dict(m=64, w=2, extra=2, bounded="all"),
    (2, "ws"): dict(m=1400, w=2, extra=0, bounded="none"),
    (4, "smem_staged"): dict(m=4, w=3),
    (4, "smem_l2"): dict(m=20, w=4, extra=20, full_span=True, bounded="none"),
    (4, "hybrid"): dict(m=96, w=4, extra=0, bounded="all"),
    (4, "ws"): dict(m=1024, w=4, extra=0, bounded="none"),
    (8, "smem_staged"): dict(m=8, w=7, bounded="none"),
    (8, "smem_l2"): dict(m=128, w=8, extra=0, bounded="none"),
    (8, "hybrid"): dict(m=32, w=8, extra=4, bounded="all"),
    (8, "ws"): dict(m=512, w=8, extra=0, bounded="none"),
    (16, "smem_staged"): dict(m=10, w=9),
    (16, "smem_l2"): dict(m=64, w=16, extra=0),
    (16, "hybrid"): dict(m=48, w=16, extra=0),
    (16, "ws"): dict(m=256, w=16, extra=0, bounded="none"),
    (32, "smem_staged"): dict(m=18, w=17, extra=0, bounded="none"),
    (32, "smem_l2"): dict(m=34, w=32, extra=0, bounded="none"),
    (32, "hybrid"): dict(m=24, w=17, extra=0, bounded="none"),
    (32, "ws"): dict(m=96, w=32, extra=0, bounded="none"),
}
# per-LP matrices (amap) in every placement: the LP's own A, A' and assembly products sit behind its band
AMAP_CASES = {
    (4, "smem_staged"): dict(m=8, w=4, extra=0, bounded="none"),
    (16, "smem_l2"): dict(m=32, w=16, extra=0, bounded="none"),
    (8, "hybrid"): dict(m=16, w=8, extra=4, bounded="mixed"),
    (2, "ws"): dict(m=192, w=2, extra=0, bounded="none"),
}
# scaled / degenerate data and column-kind edges, all on small shared-memory templates
VARIANTS = {
    "nb0": dict(m=12, w=2, bounded="none"),
    "nb_all": dict(m=12, w=2, bounded="all"),
    "c_up": dict(m=12, w=2, c_scale=2.0 ** 20),
    "c_down": dict(m=12, w=2, c_scale=2.0 ** -20),
    "b_up": dict(m=12, w=3, b_scale=2.0 ** 20),
    "b_down": dict(m=12, w=3, b_scale=2.0 ** -20),
    "u_loose": dict(m=12, w=3, bounded="all", u_scale=2.0 ** 20),
    "c_zero": dict(m=12, w=1, zero_c=True),
    "b_zero": dict(m=12, w=1, zero_b=True),
}


# ---------------------------------------------------------------------------------------------------------------------
# placement of a band-kernel launch: a mirror of band_geometry() in csrc/dsp_lp.cu (used to choose test shapes; the GPU tests
# assert the placement the library really picked, from dsp_lp_last_launch)
# ---------------------------------------------------------------------------------------------------------------------
PLACEMENTS = ("smem_staged", "smem_l2", "hybrid", "ws")


def padded_w(w):
    wt = 1
    while wt < w:
        wt *= 2
    return wt


def sizes(t: LPTemplate):
    """(W, nnz, nasm, band_doubles, prob_doubles, hot_bytes) of a finalized template as the library lays it out"""
    m, n, nb = t.m, t.n, t.nb
    W = padded_w(t.w)
    A = t.A.tocsc()
    cnt = np.diff(A.indptr)
    nnz = int(A.nnz)
    nasm = int((cnt * (cnt + 1) // 2).sum())
    band = (m + 2 * W) * (W + 2)
    prob = 8 * n + 6 * nb + 3 * m + band
    if t.amap is not None:
        band += 2 * nnz + nasm
        prob += 2 * nnz + nasm
    ints = (m + 1) + nnz + (n + 1) + nnz + (m * (W + 1) + 1) + nasm
    hot = (2 * nnz + nasm) * 8 + ints * 4
    hot = (hot + 15) // 16 * 16
    return W, nnz, nasm, band, prob, hot


def band_placement(t: LPTemplate, budget=H100_SMEM_OPTIN):
    """placement band_geometry() picks for this template: one of PLACEMENTS, and the warps per CTA before the small-batch spread"""
    W, nnz, nasm, band, prob, hot = sizes(t)
    pb, bb = prob * 8, band * 8
    off = 16 + hot
    smem_w = (budget - off) // pb if budget > off else 0
    staged = True
    if smem_w < 4:
        staged = False
        smem_w = (budget - 16) // pb
    hyb_w = min(KMAX_WARPS, (budget - 16) // bb) if bb + 16 <= budget else 0
    if smem_w >= 7 or (hyb_w < 6 and smem_w >= 4):
        return ("smem_staged" if staged else "smem_l2"), min(smem_w, KMAX_WARPS)
    if hyb_w >= 6:
        return "hybrid", hyb_w
    return "ws", KMAX_WARPS


def placement_of_launch(t: LPTemplate, launch):
    """placement a band-kernel launch ran in, from its dynamic shared memory and warps per CTA (dsp_lp_last_launch)"""
    _, _, _, band, prob, _ = sizes(t)
    warps = launch["block"] // 32
    s = launch["smem_bytes"]
    if s == 16:
        return "ws"
    if s == 16 + warps * band * 8:
        return "hybrid"
    if s == 16 + warps * prob * 8:
        return "smem_l2"
    if s > 16 + warps * prob * 8:
        return "smem_staged"
    raise AssertionError(f"unrecognised band launch {launch} (band {band}, prob {prob} doubles)")
