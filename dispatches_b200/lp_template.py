"""Shared standard-form LP template for a batch of structurally identical dispatch LPs.

One template = one (case-study flowsheet, horizon T, fixed/free design mode).  Every LP of a batch is

    min  c'x + obj_const      s.t.  A x = b,   0 <= x <= u            (u_j = +inf allowed)

with the constraint matrix ``A`` (inequality rows already carry a slack column) SHARED by the whole
batch, and the per-problem data affine in two small parameter vectors:

    c = c0 + Cmap @ cparams        (cparams: the LMP signal, what changes per price scenario)
    b = b0 + Bmap @ rparams        (rparams: capacity-factor / design scalars, what changes per design)
    u = u0 + Umap @ rparams
    obj_const = o0 + omap @ rparams

This is the data model behind the C-ABI (include/dsp_lp.h: dsp_lp_template_create) and replaces, for the
hot path, what Pyomo's LP writer + CBC's reader rebuild per LP in the reference
(wind_battery_LMP.py:195-267: model build + SolverFactory("cbc").solve per scenario).

``finalize()`` does the once-per-template symbolic work the GPU kernel relies on: a bandwidth-reducing
row order for the normal matrix  M = A D A'  (block-tridiagonal in time for every multi-period flowsheet,
SURVEY.md §0.5), the band half-width ``w`` and the assembly list  M[i, i-k] = sum_p coef_p * d[col_p].
"""
from __future__ import annotations

import dataclasses
import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import reverse_cuthill_mckee

INF = float("inf")


@dataclasses.dataclass
class LPTemplate:
    name: str
    A: sp.csr_matrix                 # m x n (slacks included)
    b0: np.ndarray
    Bmap: sp.csr_matrix              # m x Pr
    c0: np.ndarray
    Cmap: sp.csr_matrix              # n x Pc
    u0: np.ndarray                   # +inf where unbounded above
    Umap: sp.csr_matrix              # n x Pr (rows of unbounded columns are empty)
    o0: float
    omap: np.ndarray                 # Pr
    ocmap: np.ndarray                # Pc   (objective constant = o0 + omap@rparams + ocmap@cparams)
    col_shift: np.ndarray            # x_model = col_shift + col_scale * x_template   (lower-bound shift, equilibration)
    col_scale: np.ndarray
    col_names: list
    row_names: list
    meta: dict = dataclasses.field(default_factory=dict)
    # filled by finalize()
    row_perm: np.ndarray | None = None
    w: int = 0
    asm_ptr: np.ndarray | None = None
    asm_col: np.ndarray | None = None
    asm_val: np.ndarray | None = None
    # per-problem matrix coefficients: A[row, col] = A0[row, col] + sum coef * rparams[param]  (rows / cols in template order)
    amap: tuple | None = None        # (rows, cols, params, coefs) int / int / int / float arrays

    @property
    def m(self):
        return self.A.shape[0]

    @property
    def n(self):
        return self.A.shape[1]

    @property
    def Pc(self):
        return self.Cmap.shape[1]

    @property
    def Pr(self):
        return self.Bmap.shape[1]

    @property
    def nb(self):
        """number of upper-bounded columns (ordered first)."""
        return int(np.isfinite(self.u0).sum())

    # ------------------------------------------------------------------
    def instantiate(self, cparams, rparams):
        """(c, b, u, obj_const) of one problem -- host-side helper for tests / plumbing."""
        cparams = np.asarray(cparams, float); rparams = np.asarray(rparams, float)
        c = self.c0 + self.Cmap @ cparams
        b = self.b0 + self.Bmap @ rparams
        u = self.u0.copy()
        fin = np.isfinite(u)
        u[fin] = u[fin] + (self.Umap @ rparams)[fin]
        return c, b, u, self.o0 + float(self.omap @ rparams) + float(self.ocmap @ cparams)

    def matrix(self, rparams):
        """the constraint matrix of one problem (A itself when the template has no matrix parameters)"""
        if self.amap is None:
            return self.A
        r, c, k, v = self.amap
        A = self.A.tolil(copy=True)
        rparams = np.asarray(rparams, float)
        for i, j, kk, vv in zip(r, c, k, v):
            A[i, j] = A[i, j] + vv * rparams[kk]
        return A.tocsr()

    # ------------------------------------------------------------------
    def finalize(self, equilibrate=False):
        """Column order (bounded first), row order (min bandwidth of A A'), band assembly list."""
        A = self.A.tocsr()
        m, n = A.shape
        # 1. bounded columns first (keeps the upper-bound vectors short in the kernel)
        fin = np.isfinite(self.u0)
        cperm = np.concatenate([np.flatnonzero(fin), np.flatnonzero(~fin)])
        A = A[:, cperm]
        self.c0 = self.c0[cperm]; self.Cmap = self.Cmap.tocsr()[cperm]
        self.u0 = self.u0[cperm]; self.Umap = self.Umap.tocsr()[cperm]
        self.col_shift = self.col_shift[cperm]; self.col_scale = self.col_scale[cperm]
        self.col_names = [self.col_names[j] for j in cperm]
        if self.amap is not None:
            inv = np.empty(n, int); inv[cperm] = np.arange(n)
            self.amap = (self.amap[0], inv[self.amap[1]], self.amap[2], self.amap[3])
        # 1b. geometric-mean equilibration  A <- R A C  (x = C x~, b~ = R b, c~ = C c, u~ = u / C)
        if equilibrate:
            A = A.tocsr().astype(float)
            R = np.ones(m); C = np.ones(n)
            for _ in range(6):
                B = sp.diags(R) @ A @ sp.diags(C)
                B = B.tocsr(); absB = abs(B)
                rmax = absB.max(axis=1).toarray().ravel(); rmin = _rowmin(absB)
                R /= np.sqrt(np.maximum(rmax * rmin, 1e-300))
                B = (sp.diags(R) @ A @ sp.diags(C)).tocsc(); absB = abs(B)
                cmax = absB.max(axis=0).toarray().ravel(); cmin = _rowmin(absB.T.tocsr())
                C /= np.sqrt(np.maximum(cmax * cmin, 1e-300))
            # round to powers of two: scaling is then exact in floating point
            R = 2.0 ** np.round(np.log2(R)); C = 2.0 ** np.round(np.log2(C))
            A = (sp.diags(R) @ A @ sp.diags(C)).tocsr()
            self.b0 = self.b0 * R; self.Bmap = (sp.diags(R) @ self.Bmap).tocsr()
            self.c0 = self.c0 * C; self.Cmap = (sp.diags(C) @ self.Cmap).tocsr()
            self.u0 = self.u0 / C; self.Umap = (sp.diags(1.0 / C) @ self.Umap).tocsr()
            self.col_scale = self.col_scale * C
            self.meta["row_scale"] = R
            if self.amap is not None:
                self.amap = (self.amap[0], self.amap[1], self.amap[2], self.amap[3] * R[self.amap[0]] * C[self.amap[1]])
        # 2. row order: natural vs reverse Cuthill-McKee on the pattern of A A'
        P = (abs(A) @ abs(A).T).tocsr()
        P.data[:] = 1.0

        def bandwidth(perm):
            inv = np.empty(m, int); inv[perm] = np.arange(m)
            coo = P.tocoo()
            return int(np.max(np.abs(inv[coo.row] - inv[coo.col]))) if coo.nnz else 0

        nat = np.arange(m)
        rcm = np.asarray(reverse_cuthill_mckee(P, symmetric_mode=True))
        perm = nat if bandwidth(nat) <= bandwidth(rcm) else rcm
        self.w = bandwidth(perm)
        self.row_perm = perm
        A = A[perm]
        self.b0 = self.b0[perm]; self.Bmap = self.Bmap.tocsr()[perm]
        self.row_names = [self.row_names[i] for i in perm]
        if self.amap is not None:
            invr = np.empty(m, int); invr[perm] = np.arange(m)
            self.amap = (invr[self.amap[0]], self.amap[1], self.amap[2], self.amap[3])
        self.A = A.tocsr(); self.A.sort_indices()
        # 3. assembly list of the lower band of M = A D A'
        w = self.w
        Acsc = self.A.tocsc()
        ent = [[] for _ in range(m * (w + 1))]
        for j in range(n):
            lo, hi = Acsc.indptr[j], Acsc.indptr[j + 1]
            rows, vals = Acsc.indices[lo:hi], Acsc.data[lo:hi]
            for a in range(len(rows)):
                for bq in range(len(rows)):
                    i, i2 = rows[a], rows[bq]
                    if i2 <= i:
                        ent[i * (w + 1) + (i - i2)].append((j, vals[a] * vals[bq]))
        ptr = np.zeros(m * (w + 1) + 1, np.int32)
        cols, vals = [], []
        for e, lst in enumerate(ent):
            ptr[e + 1] = ptr[e] + len(lst)
            for j, v in lst:
                cols.append(j); vals.append(v)
        self.asm_ptr, self.asm_col, self.asm_val = ptr, np.array(cols, np.int32), np.array(vals, float)
        return self

    # ------------------------------------------------------------------
    def column(self, name):
        return self.col_names.index(name)


def _rowmin(absB):
    """min over the stored nonzeros of each row of a CSR matrix (rows without entries -> 1)."""
    out = np.ones(absB.shape[0])
    for i in range(absB.shape[0]):
        d = absB.data[absB.indptr[i]:absB.indptr[i + 1]]
        d = d[d > 0]
        if d.size:
            out[i] = d.min()
    return out


class TemplateBuilder:
    """Tiny algebra for writing a template: columns, (in)equality rows, parameter-affine data.

    A "parameter-affine" quantity is  const + sum_k coef_k * param[k]  given as ``(const, {k: coef})``
    or a plain float.
    """

    def __init__(self, name, Pc, Pr):
        self.name, self.Pc, self.Pr = name, Pc, Pr
        self.cols, self.rows = [], []          # names
        self.u = []                            # (const, {k: coef}) or None
        self.lbs, self.fixed = [], []          # constant lower bound ; True if the column is a constant
        self.ocmap = np.zeros(Pc)
        self.c = []                            # (const, {k: coef})
        self.arows, self.rhs = [], []          # dict col->val ; (const, {k:coef})
        self.o0, self.omap = 0.0, np.zeros(Pr)
        self.acoef = []                        # (row, col, rparam, coef): per-problem matrix coefficients
        self.meta = {}

    @staticmethod
    def _aff(q):
        if q is None:
            return None
        if isinstance(q, tuple):
            return float(q[0]), dict(q[1])
        return float(q), {}

    def var(self, name, ub=None, lb=0.0, fix=None):
        """column with lb <= x <= ub (lb constant, ub parameter-affine) or a constant (fix=value)."""
        if fix is not None:
            lb, ub = float(fix), None
        self.cols.append(name); self.u.append(self._aff(ub)); self.c.append((0.0, {}))
        self.lbs.append(float(lb)); self.fixed.append(fix is not None)
        return len(self.cols) - 1

    def cost(self, j, q):
        c0, cm = self.c[j]; a0, am = self._aff(q)
        for k, v in am.items():
            cm[k] = cm.get(k, 0.0) + v
        self.c[j] = (c0 + a0, cm)

    def eq(self, name, coeffs, rhs=0.0):
        """coefficients are floats, or ``(nominal, {k: coef})`` for an entry that varies per problem with rparams[k] (the nominal value
        keeps the entry in the sparsity pattern and is what the once-per-template scaling sees)"""
        plain = {}
        for j, v in dict(coeffs).items():
            if isinstance(v, tuple):
                plain[j] = float(v[0])
                for k, cf in v[1].items():
                    self.acoef.append((len(self.rows), j, int(k), float(cf)))
            else:
                plain[j] = v
        self.rows.append(name); self.arows.append(plain); self.rhs.append(self._aff(rhs))

    def le(self, name, coeffs, rhs=0.0):
        s = self.var("slack:" + name)
        coeffs = dict(coeffs); coeffs[s] = 1.0
        self.eq(name, coeffs, rhs)

    def obj_const(self, q):
        a0, am = self._aff(q)
        self.o0 += a0
        for k, v in am.items():
            self.omap[k] += v

    def build(self, equilibrate=False) -> LPTemplate:
        # substitute x = lb + x' (and drop constant columns)
        lbs = np.array(self.lbs)
        for r, row in enumerate(self.arows):
            shift = sum(v * lbs[j] for j, v in row.items())
            if shift != 0.0:
                a0, am = self.rhs[r]; self.rhs[r] = (a0 - shift, am)
        for j in range(len(self.cols)):
            if lbs[j] != 0.0:
                c0, cm = self.c[j]
                self.o0 += c0 * lbs[j]
                for k, v in cm.items():
                    self.ocmap[k] += v * lbs[j]
                if self.u[j] is not None:
                    u0, um = self.u[j]; self.u[j] = (u0 - lbs[j], um)
        keep = [j for j in range(len(self.cols)) if not self.fixed[j]]
        remap = {j: k for k, j in enumerate(keep)}
        self.arows = [{remap[j]: v for j, v in row.items() if j in remap} for row in self.arows]
        self.cols = [self.cols[j] for j in keep]; self.u = [self.u[j] for j in keep]
        self.c = [self.c[j] for j in keep]; shifts = lbs[keep]
        n, m = len(self.cols), len(self.rows)

        def affine_rows(items, P, default=0.0):
            base = np.full(len(items), default)
            ri, ci, vv = [], [], []
            for r, it in enumerate(items):
                if it is None:
                    continue
                base[r] = it[0]
                for k, v in it[1].items():
                    ri.append(r); ci.append(k); vv.append(v)
            return base, sp.csr_matrix((vv, (ri, ci)), shape=(len(items), P))

        ri, ci, vv = [], [], []
        for r, row in enumerate(self.arows):
            for j, v in row.items():
                if v != 0.0:
                    ri.append(r); ci.append(j); vv.append(v)
        A = sp.csr_matrix((vv, (ri, ci)), shape=(m, n))
        b0, Bmap = affine_rows(self.rhs, self.Pr)
        c0, Cmap = affine_rows(self.c, self.Pc)
        u0, Umap = affine_rows(self.u, self.Pr, default=INF)
        t = LPTemplate(self.name, A, b0, Bmap, c0, Cmap, u0, Umap, self.o0, self.omap.copy(), self.ocmap.copy(),
                       shifts.copy(), np.ones(n), list(self.cols), list(self.rows), dict(self.meta))
        if self.acoef:
            for r, j, k, cf in self.acoef:
                if lbs[j] != 0.0 or j not in remap:
                    raise ValueError("a per-problem matrix coefficient needs a free-standing column with lower bound 0")
            t.amap = (np.array([a[0] for a in self.acoef], int), np.array([remap[a[1]] for a in self.acoef], int),
                      np.array([a[2] for a in self.acoef], int), np.array([a[3] for a in self.acoef], float))
        return t.finalize(equilibrate=equilibrate)


# ----------------------------------------------------------------------------------------------------------------------
def standard_form(rows, lo, hi, lb, ub, cost, c0=0.0, sense=1.0, var_names=None, row_names=None, name="lp",
                  p0=None, dcost=None, dlo=None, dhi=None, dlb=None, dub=None, dc0=None, equilibrate=True, presolve=True):
    """General LP -> LPTemplate (the pure, pyomo-free half of the Pyomo walker; SURVEY.md 8(f)-1).

        optimise  sense * (cost'x + c0)   s.t.   lo <= rows x <= hi,   lb <= x <= ub

    ``rows`` is a list of {column: coefficient} dicts; any of lo / hi / lb / ub may be -inf / +inf (free Vars such as
    pem.electricity -- domain Reals, unit_models/pem_electrolyzer.py:96-100 -- ranged rows, fixed Vars lb == ub).
    Batched parameters: the LP was extracted at parameter values ``p0`` [P]; ``dcost`` [n,P], ``dlo`` / ``dhi`` [m,P],
    ``dlb`` / ``dub`` [n,P], ``dc0`` [P] are the derivatives of the affine data with respect to them (the constraint matrix
    may not depend on parameters: it is shared by the batch).  One parameter vector serves as cparams and rparams.

    Column transformations (undone by ``model_values``):  fixed -> constant;  finite lb: x = lb + x';  only ub finite:
    x = ub - x';  free: x = x+ - x-;  both finite: 0 <= x' <= ub - lb.  Inequality rows get a slack column, ranged rows a bounded
    one.  ``presolve`` substitutes doubleton equalities  a x_i + b x_j = rhs  with a free / identically bounded x_i (the arcs and
    link constraints of a Pyomo multi-period model, wind_battery_LMP.py:22-50) -- they would otherwise widen the band of A A'.
    Returns an LPTemplate whose meta["recover"] maps template columns back to the model's variables and meta["row_of"] the
    template row of every model row (for duals)."""
    n = len(lb)
    m = len(rows)
    lb = np.asarray(lb, float).copy(); ub = np.asarray(ub, float).copy()
    lo = np.asarray(lo, float).copy(); hi = np.asarray(hi, float).copy()
    P = 0 if p0 is None else len(p0)
    p0 = np.zeros(0) if p0 is None else np.asarray(p0, float)
    Z = lambda a, shape: np.zeros(shape) if a is None else np.asarray(a, float).reshape(shape)
    dcost, dlo, dhi, dlb, dub, dc0 = Z(dcost, (n, P)), Z(dlo, (m, P)), Z(dhi, (m, P)), Z(dlb, (n, P)), Z(dub, (n, P)), Z(dc0, (P,))
    cvec = np.zeros(n)
    for j, v in (cost.items() if isinstance(cost, dict) else enumerate(np.asarray(cost, float))):
        cvec[j] = v
    # ---- model variable j = const_j + sum_k coef * y_k in terms of working variables y (affine in params through const)
    # working representation: every model variable is  shift_j(p) + sign_j * y_{col_j}  [- y_{col2_j}] ; presolve may alias
    # variable i to variable j:  x_i = alpha * x_j + beta
    alias = {}                                        # i -> (j, alpha, beta0, dbeta[P])
    elim = []                                         # (e, row, a_e, cost_e, dcost_e, {other live row: coef of e}), in elimination order
    rows = [dict(r) for r in rows]
    model = dict(rows=[dict(r) for r in rows], cost=cvec.copy(), dcost=dcost.copy())
    live_row = np.ones(m, bool)
    if presolve:
        use = [set() for _ in range(n)]
        for r, row in enumerate(rows):
            for j in row:
                use[j].add(r)
        changed = True
        while changed:
            changed = False
            for r in range(m):
                if not live_row[r] or lo[r] != hi[r] or len(rows[r]) != 2 or np.any(dlo[r] != dhi[r]):
                    continue
                (i, a), (j, b) = rows[r].items()
                fixed = lambda k: lb[k] == ub[k] and not dlb[k].any() and not dub[k].any()
                if fixed(i) or fixed(j):
                    continue
                # eliminate the one whose bounds are implied: free, or the same box after the affine map (alpha > 0, beta = 0)
                for (e, ae), (k, ak) in (((i, a), (j, b)), ((j, b), (i, a))):
                    alpha, beta = -ak / ae, hi[r] / ae
                    same_box = alpha == 1.0 and beta == 0.0 and not dhi[r].any() and lb[e] == lb[k] and ub[e] == ub[k] \
                        and not (dlb[e] - dlb[k]).any() and not (dub[e] - dub[k]).any()
                    free = not np.isfinite(lb[e]) and not np.isfinite(ub[e])
                    if not (free or same_box) or dcost[e].any() and (dhi[r].any()):
                        continue
                    # merging must stay local in time: chains of link equalities over ALL periods (nameplate_power[t] =
                    # nameplate_power[t+1]) would collapse into one dense column and destroy the band of A A'
                    if len((use[e] | use[k]) - {r}) > 8:
                        continue
                    # substitute x_e = alpha x_k + beta(p) everywhere
                    alias[e] = (k, alpha, beta, dhi[r] / ae)
                    elim.append((e, r, ae, cvec[e], dcost[e].copy(),
                                 {rr: rows[rr][e] for rr in use[e] if rr != r and live_row[rr] and e in rows[rr]}))
                    live_row[r] = False
                    for rr in list(use[e]):
                        if rr == r or not live_row[rr]:
                            continue
                        coef = rows[rr].pop(e)
                        rows[rr][k] = rows[rr].get(k, 0.0) + coef * alpha
                        if rows[rr][k] == 0.0:
                            del rows[rr][k]
                        else:
                            use[k].add(rr)
                        lo[rr] -= coef * beta; hi[rr] -= coef * beta
                        dlo[rr] = dlo[rr] - coef * dhi[r] / ae; dhi[rr] = dhi[rr] - coef * dhi[r] / ae
                    c0 = c0 + cvec[e] * beta
                    dc0 = dc0 + cvec[e] * dhi[r] / ae + dcost[e] * beta
                    cvec[k] += cvec[e] * alpha; dcost[k] = dcost[k] + dcost[e] * alpha
                    cvec[e] = 0.0; dcost[e] = 0.0
                    use[e] = set()
                    changed = True
                    break
    # ---- columns
    kind = np.zeros(n, int)          # 0 fixed/const, 1 lb-shift, 2 ub-flip, 3 free split, 4 boxed, 5 alias
    col, col2 = -np.ones(n, int), -np.ones(n, int)
    cols_u0, cols_du, names = [], [], []
    vn = var_names or [f"x[{j}]" for j in range(n)]
    nc = 0
    for j in range(n):
        if j in alias:
            kind[j] = 5
            continue
        moving = dlb[j].any() or dub[j].any()
        if lb[j] == ub[j] and not moving:
            kind[j] = 0
        elif np.isfinite(lb[j]) and np.isfinite(ub[j]):
            kind[j] = 4; col[j] = nc; nc += 1; cols_u0.append(ub[j] - lb[j]); cols_du.append(dub[j] - dlb[j]); names.append(vn[j])
        elif np.isfinite(lb[j]):
            kind[j] = 1; col[j] = nc; nc += 1; cols_u0.append(INF); cols_du.append(np.zeros(P)); names.append(vn[j])
        elif np.isfinite(ub[j]):
            kind[j] = 2; col[j] = nc; nc += 1; cols_u0.append(INF); cols_du.append(np.zeros(P)); names.append(vn[j] + ":flipped")
        else:
            kind[j] = 3; col[j] = nc; col2[j] = nc + 1; nc += 2
            cols_u0 += [INF, INF]; cols_du += [np.zeros(P)] * 2; names += [vn[j] + ":pos", vn[j] + ":neg"]
    # x_j = shift_j(p) + sgn_j * y[col_j] (- y[col2_j])
    shift0 = np.where(kind == 2, ub, np.where((kind == 1) | (kind == 4) | (kind == 0), lb, 0.0))
    shift0 = np.where(np.isfinite(shift0), shift0, 0.0)
    dshift = np.where((kind == 2)[:, None], dub, np.where(((kind == 1) | (kind == 4))[:, None], dlb, 0.0))
    sgn = np.where(kind == 2, -1.0, 1.0)
    if np.any((np.abs(dcost).sum(1) > 0) & (np.abs(dshift).sum(1) > 0)):
        raise ValueError("a Var whose cost AND whose bound depend on batched Params makes the objective constant quadratic in them")
    # ---- rows
    ri, ci, vv = [], [], []
    b0, db, row_of = [], [], -np.ones(m, int)
    slack_sign = []
    mr = 0
    for r in range(m):
        if not live_row[r]:
            continue
        row = rows[r]
        if not any(kind[j] != 0 for j in row):       # only constants left (fixed Vars): nothing to solve for in this row
            continue
        sh = sum(a * shift0[j] for j, a in row.items()); dsh = sum(a * dshift[j] for j, a in row.items())
        for j, a in row.items():
            if kind[j] == 0:
                continue
            ri.append(mr); ci.append(col[j]); vv.append(a * sgn[j])
            if kind[j] == 3:
                ri.append(mr); ci.append(col2[j]); vv.append(-a)
        if lo[r] == hi[r] and not (dlo[r] - dhi[r]).any():
            b0.append(hi[r] - sh); db.append(dhi[r] - dsh)
        elif not np.isfinite(lo[r]):
            ri.append(mr); ci.append(nc); vv.append(1.0); nc += 1
            cols_u0.append(INF); cols_du.append(np.zeros(P)); names.append(f"slack[{r}]")
            b0.append(hi[r] - sh); db.append(dhi[r] - dsh)
        elif not np.isfinite(hi[r]):
            ri.append(mr); ci.append(nc); vv.append(-1.0); nc += 1
            cols_u0.append(INF); cols_du.append(np.zeros(P)); names.append(f"surplus[{r}]")
            b0.append(lo[r] - sh); db.append(dlo[r] - dsh)
        else:                                         # ranged: a x + s = hi, 0 <= s <= hi - lo
            ri.append(mr); ci.append(nc); vv.append(1.0); nc += 1
            cols_u0.append(hi[r] - lo[r]); cols_du.append(dhi[r] - dlo[r]); names.append(f"range[{r}]")
            b0.append(hi[r] - sh); db.append(dhi[r] - dsh)
        row_of[r] = mr
        mr += 1
    A = sp.csr_matrix((vv, (ri, ci)), shape=(mr, nc))
    A.sum_duplicates()
    # ---- objective: sense * (sum_j c_j(p) x_j + c0(p)),  x_j = shift_j(p) + sgn_j y  (cost or shift param-free per column)
    c_t = np.zeros(nc); C_t = np.zeros((nc, P))
    for j in range(n):
        if kind[j] in (0, 5):
            continue
        c_t[col[j]] += sense * cvec[j] * sgn[j]; C_t[col[j]] += sense * dcost[j] * sgn[j]
        if kind[j] == 3:
            c_t[col2[j]] -= sense * cvec[j]; C_t[col2[j]] -= sense * dcost[j]
    o_at_p0 = sense * (c0 + float(cvec @ shift0))
    do = sense * (dc0 + dcost.T @ shift0 + dshift.T @ cvec)
    b0 = np.array(b0, float); db = np.array(db, float).reshape(mr, P)
    u0 = np.array(cols_u0, float); dU = np.array(cols_du, float).reshape(nc, P)
    # values at p0 -> affine maps in p:  q(p) = q(p0) + dq (p - p0)
    t = LPTemplate(name, A, b0 - db @ p0 if P else b0, sp.csr_matrix(db), c_t - C_t @ p0 if P else c_t, sp.csr_matrix(C_t),
                   np.where(np.isfinite(u0), u0 - (dU @ p0 if P else 0.0), INF), sp.csr_matrix(np.where(np.isfinite(u0)[:, None], dU, 0.0)),
                   o_at_p0 - float(do @ p0) if P else o_at_p0, do.copy() * 0.0, do.copy(),
                   np.zeros(nc), np.ones(nc), names, [f"row[{i}]" for i in range(mr)],
                   dict(kind="standard_form", sense=sense))
    t.meta["recover"] = dict(kind=kind, col=col, col2=col2, sgn=sgn, shift0=shift0, dshift=dshift, p0=p0, alias=alias, names=list(names),
                             elim=elim)
    t.meta["model"] = model
    t.meta["row_of"] = row_of
    t.meta["live_row"] = live_row
    # objective constant rides on ocmap (cparams) only: omap stays zero so that cparams == rparams does not count it twice
    return t.finalize(equilibrate=equilibrate)


def model_values(t: LPTemplate, x, params=None):
    """Template-space primal x [N, n] of a standard_form() template -> the model's variable values [N, n_model]."""
    rec = t.meta["recover"]
    x = np.atleast_2d(np.asarray(x, float))
    N = x.shape[0]
    pos = {nm: k for k, nm in enumerate(t.col_names)}                  # finalize() permutes columns: go through the names
    xm = x * t.col_scale + t.col_shift
    P = rec["p0"].size
    dp = (np.atleast_2d(params) - rec["p0"]) if (params is not None and P) else np.zeros((N, P))
    n = rec["kind"].size
    out = np.zeros((N, n))
    names = rec["names"]
    for j in range(n):
        k = rec["kind"][j]
        if k == 5:
            continue
        v = rec["shift0"][j] + (dp @ rec["dshift"][j] if P else 0.0)
        if k != 0:
            v = v + rec["sgn"][j] * xm[:, pos[names[rec["col"][j]]]]
            if k == 3:
                v = v - xm[:, pos[names[rec["col2"][j]]]]
        out[:, j] = v
    done = set(j for j in range(n) if rec["kind"][j] != 5)
    pending = dict(rec["alias"])
    while pending:                                                      # aliases may chain
        for e, (k, alpha, beta, dbeta) in list(pending.items()):
            if k in done:
                out[:, e] = alpha * out[:, k] + beta + (dp @ dbeta if P else 0.0)
                done.add(e); del pending[e]
    return out


def model_duals(t: LPTemplate, y):
    """Row duals y [N, m] of a standard_form() template -> d(objective)/d(rhs) of the model's rows [N, m_model] (0 for rows
    presolve removed)."""
    y = np.atleast_2d(np.asarray(y, float))
    R = t.meta.get("row_scale")
    pos = {nm: k for k, nm in enumerate(t.row_names)}
    row_of = t.meta["row_of"]
    out = np.zeros((y.shape[0], row_of.size))
    for r, mr in enumerate(row_of):
        if mr >= 0:
            k = pos[f"row[{mr}]"]
            out[:, r] = y[:, k] * (R[mr] if R is not None else 1.0) * t.meta["sense"]
    return out


def model_reduced_costs(t: LPTemplate, y, params=None):
    """Reduced costs of the model's variables [N, n_model] of a standard_form() template from its row duals y [N, m]:
    rc = c_model(params) - A_model' y_model, in the model's own objective sense, with y_model the duals of model_duals() and, for the rows
    presolve removed, the duals that make each eliminated variable's reduced cost 0 (solved back in reverse elimination order; a free
    variable has reduced cost 0 at every optimum, and for a variable merged with an identically bounded one that choice leaves the
    bound multipliers on the one kept).  Fixed, flipped, split and presolved variables are then covered by the definition itself."""
    rec, mdl = t.meta["recover"], t.meta["model"]
    ym = model_duals(t, y)
    N, n = ym.shape[0], rec["kind"].size
    P = rec["p0"].size
    dp = (np.atleast_2d(params) - rec["p0"]) if (params is not None and P) else np.zeros((N, P))
    for e, r, ae, ce, dce, others in reversed(rec["elim"]):
        c_e = ce + (dp @ dce if P else 0.0)
        ym[:, r] = (c_e - sum(a * ym[:, rr] for rr, a in others.items())) / ae
    ri, ci, vv = [], [], []
    for r, row in enumerate(mdl["rows"]):
        for j, a in row.items():
            ri.append(r); ci.append(j); vv.append(a)
    A = sp.csr_matrix((vv, (ri, ci)), shape=(len(mdl["rows"]), n))
    c = mdl["cost"][None, :] + (dp @ mdl["dcost"].T if P else 0.0)
    return c - (A.T @ ym.T).T


# ----------------------------------------------------------------------------------------------------------------------
def detect_chain1(t: LPTemplate, max_flows=3):
    """Structure recognition for the descriptor-driven "single storage chain" stage kernel (csrc/dsp_stage_chain1.cuh):
    every column of the template appears in ONE row (a flow of that period) or in TWO rows that are neighbours in a simple path
    through all rows (the state carried from one period to the next), at most one state per period and ``max_flows`` flows.
    Returns None when the template is not of that family, else dict(T, NF, col_idx [T, NF+1], row_idx [T], coef [T, NF+1],
    coef_next [T]) in template (equilibrated) units -- the kernel needs nothing else that is flowsheet specific."""
    A = t.A.tocsc()
    m, n = A.shape
    cnt = np.diff(A.indptr)
    if m < 2 or np.any(cnt < 1) or np.any(cnt > 2):
        return None
    nbr = [dict() for _ in range(m)]                  # row -> {neighbour row: state column}
    flows = [[] for _ in range(m)]
    for j in range(n):
        rows = A.indices[A.indptr[j]:A.indptr[j + 1]]
        if len(rows) == 1:
            flows[rows[0]].append(j)
        else:
            a, b = int(rows[0]), int(rows[1])
            if b in nbr[a]:
                return None                           # two states between the same pair of periods: K = 2 family
            nbr[a][b] = j; nbr[b][a] = j
    deg = np.array([len(d) for d in nbr])
    if np.any(deg > 2):
        return None
    ends = np.flatnonzero(deg <= 1)
    if len(ends) != 2:
        return None                                   # a cycle (periodic storage) or several chains
    order, prev, cur = [], -1, int(ends.min())
    while True:
        order.append(cur)
        nxt = [r for r in nbr[cur] if r != prev]
        if not nxt:
            break
        prev, cur = cur, nxt[0]
    if len(order) != m:
        return None
    T = m
    # the last period has no successor: its state slot is free and may hold one of its single-row columns
    NF = max([2] + [len(flows[r]) for r in order[:-1]] + [len(flows[order[-1]]) - 1])
    if NF > max_flows:
        return None
    Acsr = t.A.tocsr()
    col_idx = -np.ones((T, NF + 1), np.int32); coef = np.zeros((T, NF + 1)); coef_next = np.zeros(T)
    for k, r in enumerate(order):
        fl = list(flows[r])
        if k + 1 < T:
            j = nbr[r][order[k + 1]]
            col_idx[k, NF] = j; coef[k, NF] = Acsr[r, j]; coef_next[k] = Acsr[order[k + 1], j]
        elif len(fl) > NF or fl:
            j = fl.pop()                              # e.g. the final tank holdup
            col_idx[k, NF] = j; coef[k, NF] = Acsr[r, j]
        for f, j in enumerate(fl):
            col_idx[k, f] = j; coef[k, f] = Acsr[r, j]
    return dict(T=T, NF=int(NF), col_idx=col_idx, row_idx=np.array(order, np.int32), coef=coef, coef_next=coef_next)


# ----------------------------------------------------------------------------------------------------------------------
MAX_HALF_BANDWIDTH = 32              # widest band of A A' the band kernels are instantiated for
MAX_LINKING_COLUMNS = 8


def find_linking_columns(A, max_w=MAX_HALF_BANDWIDTH, max_k=MAX_LINKING_COLUMNS):
    """Linking columns of a constraint matrix whose A A' is too wide for the band kernels: scalar columns (a design size, a capacity)
    that sit in a row of every period.  Greedy: set aside the column with the most nonzeros, recompute the half bandwidth of the rest
    (natural vs reverse Cuthill-McKee row order, as ``finalize``), and stop as soon as it is <= max_w.

    Returns (cols, row_perm, w): the linking columns (sorted), the row order of the rest and its half bandwidth.  ``cols`` is empty
    when A A' already fits (row_perm, w are then finalize's) or when more than max_k columns would be needed (w is then the full one)."""
    A = abs(sp.csc_matrix(A))
    m, n = A.shape

    def order(keep):
        P = (A[:, keep] @ A[:, keep].T).tocsr()
        P.data[:] = 1.0
        coo = P.tocoo()

        def bw(perm):
            inv = np.empty(m, int); inv[perm] = np.arange(m)
            return int(np.max(np.abs(inv[coo.row] - inv[coo.col]))) if coo.nnz else 0
        nat = np.arange(m)
        rcm = np.asarray(reverse_cuthill_mckee(P, symmetric_mode=True))
        return (nat, bw(nat)) if bw(nat) <= bw(rcm) else (rcm, bw(rcm))

    keep = np.ones(n, bool)
    perm, w = order(keep)
    full = (perm, w)
    if w <= max_w:
        return np.zeros(0, int), perm, w
    cnt = np.diff(A.indptr)
    for _ in range(max_k):
        keep[int(np.argmax(np.where(keep, cnt, -1)))] = False
        perm, w = order(keep)
        if w <= max_w:
            return np.flatnonzero(~keep), perm, w
    return np.zeros(0, int), full[0], full[1]
