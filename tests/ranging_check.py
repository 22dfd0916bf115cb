"""The checks of ranging results (dsp_lp_ranging) on certified sets of real_lps, shared by the CPU (emulator) and GPU tests (test
infrastructure, no GPU)."""
from __future__ import annotations

import math

import numpy as np

import exact_lp as E
import exact_ranging as XR

THETA_REL = 1e-8     # kernel theta against the exact theta of the same rules, relative to |theta*| (0 and +-inf exactly)
PRED_REL = 1e-9      # the exact optimum inside the range against obj + dobj theta + d2obj theta^2 / 2, relative to max(1, |obj|)
MIRROR_REL = 1e-8    # kernel against the numpy mirror (finite values), relative to max(1e-12, |mirror|)


def directions(t, per_side=6, seed=0):
    """a sample of the coordinate axes (up to per_side cparams and per_side rparams, spread over each) plus one direction moving a
    cparam and an rparam together (d2obj != 0 where both act) -> (dir_c [K,Pc], dir_r [K,Pr], names)"""
    rows_c, rows_r, names = [], [], []
    for q in np.unique(np.linspace(0, t.Pc - 1, min(per_side, t.Pc)).astype(int)) if t.Pc else []:
        e = np.zeros(t.Pc); e[q] = 1.0
        rows_c.append(e); rows_r.append(np.zeros(t.Pr)); names.append(("c", int(q)))
    for q in np.unique(np.linspace(0, t.Pr - 1, min(per_side, t.Pr)).astype(int)) if t.Pr else []:
        e = np.zeros(t.Pr); e[q] = 1.0
        rows_c.append(np.zeros(t.Pc)); rows_r.append(e); names.append(("r", int(q)))
    if t.Pc and t.Pr:
        rng = np.random.default_rng(seed)
        gc, gr = np.zeros(t.Pc), np.zeros(t.Pr)
        gc[rng.integers(t.Pc)] = 1.0; gr[rng.integers(t.Pr)] = 0.5
        rows_c.append(gc); rows_r.append(gr); names.append(("cr", -1))
    K = len(names)
    return np.array(rows_c, float).reshape(K, t.Pc), np.array(rows_r, float).reshape(K, t.Pr), names


def against_mirror(s, basis, out, dir_c, dir_r, what=""):
    """every LP's ranges against oracle/ranging_numpy.py on the same basis: statuses equal, NaN where the mirror has NaN, finite values
    within MIRROR_REL.  Returns the (LP, direction) pairs where a ratio test met a near tie (a side 0 or +-inf in one, finite in the
    other), which the caller names."""
    from oracle import ranging_numpy as RN
    ties = []
    for k in range(len(s)):
        mr = RN.ranging(s.t, s.cparams[k], s.rparams[k], basis[0][k], basis[1][k], dir_c, dir_r)
        assert out["status"][k] == mr["status"], (what, k, out["status"][k], mr["status"])
        for f in ("lo", "hi", "dobj", "d2obj"):
            a, b = out[f][k], mr[f]
            assert np.array_equal(np.isnan(a), np.isnan(b)), (what, k, f)
            ok = ~np.isnan(b)
            both = ok & np.isfinite(b) & np.isfinite(a) & ((a == 0) == (b == 0))
            diff = ok & ~both & (a != b)
            if f in ("dobj", "d2obj"):
                scale = np.maximum(1.0, np.abs(b))
                assert (np.abs(a - b)[ok] <= 1e-9 * scale[ok]).all(), (what, k, f, np.abs(a - b)[ok].max())
                continue
            ties += [(k, int(q), f) for q in np.flatnonzero(diff)]
            rel = np.abs(a[both] - b[both]) / np.maximum(1e-12, np.abs(b[both]))
            assert (rel <= MIRROR_REL).all(), (what, k, f, rel.max())
    return ties


def exact_checks(s, k, basis, lo, hi, dobj, d2obj, dir_c, dir_r, what=""):
    """one LP and one direction against exact arithmetic, for an LP whose basis verifies exactly at theta = 0: theta against
    exact_ranging.exact_range; at theta/2 (or +-10 max(1, |p|) on an unbounded side) the basis verifies and the exact optimum equals the
    prediction; just past each finite side it does not verify.  Returns the relative theta error reached."""
    t = s.t
    cp, rp = s.cparams[k], s.rparams[k] if t.Pr else None
    obj0 = XR.verify(t, cp, rp, basis)
    elo, ehi = XR.exact_range(t, cp, rp, basis, dir_c, dir_r)
    worst = 0.0
    for got, want in ((lo, elo), (hi, ehi)):
        if want == 0.0 or math.isinf(want):
            assert got == want, (what, k, got, want)
        else:
            worst = max(worst, abs(got - want) / abs(want))
    assert worst <= THETA_REL, (what, k, lo, hi, elo, ehi)
    p = max([1.0] + [abs(float(v)) for v in np.concatenate([np.atleast_1d(cp)[np.asarray(dir_c) != 0] if t.Pc else [],
                                                             np.atleast_1d(rp)[np.asarray(dir_r) != 0] if t.Pr else []])])
    for sign, side in ((-1.0, lo), (1.0, hi)):
        th = 0.5 * side if math.isfinite(side) else sign * 10.0 * p
        if th != 0.0:
            c2, r2 = XR.moved(t, cp, rp, dir_c, dir_r, th)
            obj = float(XR.verify(t, c2, r2, basis))
            pred = float(obj0) + dobj * th + 0.5 * d2obj * th * th
            assert abs(obj - pred) <= PRED_REL * max(1.0, abs(obj)), (what, k, th, obj, pred)
        if math.isfinite(side):
            past = side + sign * 1e-6 * max(abs(side), p)
            c3, r3 = XR.moved(t, cp, rp, dir_c, dir_r, past)
            u3 = t.instantiate(c3, r3 if r3 is not None else np.zeros(0))[2]
            if ((u3 < 0) & (t.instantiate(cp, rp if rp is not None else np.zeros(0))[2] >= 0)).any():
                # the side where an upper bound reaches 0: past it the LP has no feasible point, so no basis is optimal there (the
                # kernels clip a negative bound to 0, the LP verify() checks, on which the basis can stay optimal)
                continue
            try:
                XR.verify(t, c3, r3, basis)
            except E.NotCertified:
                pass
            else:
                raise AssertionError((what, k, "the basis is still optimal past the range", side, past))
    return worst
