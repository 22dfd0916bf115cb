"""The checks of a crossover's vertices (dsp_lp_crossover) on certified sets of real_lps, shared by the CPU (emulator) and GPU tests
(test infrastructure, no GPU)."""
from __future__ import annotations

from fractions import Fraction

import numpy as np
import pytest

import exact_lp as E

OBJ_REL = 1e-9        # vertex objective against the exact optimum, relative to max(1, |obj*|)
X_REL = 1e-9          # vertex x against x* where x* is unique, relative to max(1, |x*|_inf)

# LPs whose returned basis is primal infeasible in exact arithmetic by rounding (a degenerate basic variable whose exact value is
# about -1e-12 at a primal scale of 6.4e6, one part in 1e18): like HiGHS' own bases on these LPs, they are certified after
# exact_lp._repair, whose pivot count is pinned.  {set: {LP index: repair pivots}}; every other LP verifies as it is.
PINNED = {
    "solar_battery_pem": {0: 4, 3: 2},
}


def interior_xy(s, dense=False):
    """(status, x, y) of the numpy interior-point mirror of the set's kernel family, one LP per row"""
    from oracle import ipm_dense_numpy as D, ipm_numpy as IPM
    t = s.t
    rho = t.meta.get("reg_primal", 1e-8)
    st, xs, ys = [], [], []
    for k in range(len(s)):
        c, b, u, _ = t.instantiate(s.cparams[k], s.rparams[k])
        A = t.matrix(s.rparams[k]).toarray()
        with np.errstate(all="ignore"):
            r = D.solve_batch(A, b[None], c[None], u[None], rho=rho) if dense else IPM.solve_batch(A, b[None], c[None], u[None], rho=rho)
        st.append(int(np.atleast_1d(r["status"])[0])); xs.append(np.atleast_2d(r["x"])[0]); ys.append(np.atleast_2d(r["y"])[0])
    return np.array(st, np.int32), np.array(xs), np.array(ys)


def check_vertices(s, v, status_in, pinned=None, what=""):
    """every LP crossed over OPTIMAL; its basis verifies as an exact optimum as it is (pinned LPs: after exact_lp._repair, with the
    pinned pivot count); the objective matches the exact optimum and x matches x* where that is unique.  Returns the pivot counts."""
    pinned = pinned or {}
    ok_in = status_in == 0
    assert (v["status"][ok_in] == 0).all(), (what, v["status"])
    repaired = {}
    for k in np.flatnonzero(ok_in):
        basis = (v["col_status"][k].astype(np.int8), v["row_basic"][k].astype(bool))
        assert set(np.unique(basis[0])) <= {0, 1, 2}
        assert (basis[0] == 1).sum() + basis[1].sum() == s.t.m
        if k in pinned:
            with pytest.raises(E.NotCertified):
                E.exact_optimum(s.t, s.cparams[k], s.rparams[k], basis=basis)
            repaired[int(k)] = _repair_pivots(s, k, basis)
            continue
        e = E.exact_optimum(s.t, s.cparams[k], s.rparams[k], basis=basis)
        assert abs(e.obj - s.obj[k]) <= OBJ_REL * max(1.0, abs(s.obj[k])), (what, k, e.obj, s.obj[k])
        assert np.abs(v["x"][k] - e.x).max() <= X_REL * max(1.0, np.abs(e.x).max()), (what, k)
        if s.unique_x[k]:
            assert np.abs(v["x"][k] - s.x[k]).max() <= X_REL * max(1.0, np.abs(s.x[k]).max()), (what, k)
    assert abs(v["obj"][ok_in] - s.obj[ok_in]).max() <= OBJ_REL * np.maximum(1.0, np.abs(s.obj[ok_in])).max(), what
    assert repaired == pinned, (what, repaired)
    return v["pivots"][ok_in]


def _repair_pivots(s, k, basis):
    """exact_lp._repair from the given basis: the pivots it takes to reach a basis that verifies (which it then does, as it is)"""
    t = s.t
    c, b, u, _ = t.instantiate(s.cparams[k], s.rparams[k])
    A = t.matrix(s.rparams[k]).tocsc(copy=True)
    A.sort_indices()
    fin = np.isfinite(u)
    cF, bF = E._fr(c), E._fr(b)
    uF = [Fraction(float(a)) if f else None for a, f in zip(u, fin)]
    cols = [(A.indices[A.indptr[j]:A.indptr[j + 1]], E._fr(A.data[A.indptr[j]:A.indptr[j + 1]])) for j in range(t.n)]
    col, rb = basis
    vert = E._vertex(cols, cF, bF, uF, col, rb)
    scale = max(1.0, float(np.abs(b).max(initial=0.0)), float(np.abs(u[fin]).max(initial=0.0)))
    col2, rb2, (_, _, _, rF), piv = E._repair(cols, cF, bF, uF, col, rb, vert, scale)
    zero_u = np.array([a is not None and a == 0 for a in uF])      # a fixed column the repair left at 0 goes where r_j asks
    col2 = np.where((col2 == 0) & zero_u & np.array([r < 0 for r in rF]), 2, col2).astype(np.int8)
    e = E.exact_optimum(t, s.cparams[k], s.rparams[k], basis=(col2, rb2))
    assert abs(e.obj - s.obj[k]) <= OBJ_REL * max(1.0, abs(s.obj[k]))
    return piv
