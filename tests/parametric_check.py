"""The checks of parametric walks (dsp_lp_parametric) against exact arithmetic, shared by the CPU (emulator) and GPU tests (test
infrastructure, no GPU): the log replays to bases that verify exactly on every segment, the predicted objective is the exact optimum,
every breakpoint is the exact end of the previous segment's range, and the curve is continuous and convex / concave."""
from __future__ import annotations

import math

import numpy as np

import exact_lp as E
import exact_ranging as XR

OBJ_REL = 1e-9       # predicted objective against the exact optimum, relative to max(1, |obj|)
THETA_REL = 1e-8     # a breakpoint against theta + the exact range of the previous segment's basis, relative to max(1, |theta|)
FIELDS = ("theta", "obj", "dobj", "d2obj", "enter", "leave", "leave_to", "count", "status")


def replay(t, basis, walk):
    """the basis of every event's segment: the start basis (col [n] int8, row_basic [m] bool) with events 1 .. count-1 applied in order.
    An event with enter >= 0 is a pivot (enter >= n: the artificial of row enter - n), one with enter = -1 and leave >= 0 a bound flip;
    enter = leave = -1 after event 0 ends an INFEASIBLE / UNBOUNDED walk and changes nothing."""
    col, rb = np.array(basis[0], np.int8), np.array(basis[1], bool)
    out = [(col.copy(), rb.copy())]
    n = t.n
    for e in range(1, int(walk["count"])):
        en, lv, lt = int(walk["enter"][e]), int(walk["leave"][e]), int(walk["leave_to"][e])
        if en >= 0:
            if en < n:
                col[en] = 1
            else:
                rb[en - n] = True
        if lv >= 0:
            if lv < n:
                col[lv] = 2 if lt == 2 else 0
            else:
                rb[lv - n] = False
        out.append((col.copy(), rb.copy()))
    return out


def _p(t, cp, rp, dir_c, dir_r):
    """max(1, |p|) over the parameters the direction moves"""
    vals = []
    if t.Pc and dir_c is not None:
        vals += list(np.abs(np.asarray(cp, float)[np.asarray(dir_c) != 0]))
    if t.Pr and dir_r is not None:
        vals += list(np.abs(np.asarray(rp, float)[np.asarray(dir_r) != 0]))
    return max([1.0] + vals)


def check_walk(t, cp, rp, basis, walk, dir_c, dir_r, theta_end=math.inf, events=True, exact_bases=True, what=""):
    """one walk (the fields of one (LP, direction) pair, [S] each) of an LP whose start basis verifies exactly: every segment's basis
    verifies at its midpoint (and 10 max(1, |p|) past the last event of a walk that ends OPTIMAL at +inf) with the exact objective
    equal to the prediction; every breakpoint equals theta + the exact range of the previous segment's basis; the curve is continuous.
    events: also the exact optimum (exact_lp.exact_optimum) at every event.  exact_bases=False (the dense design LPs, whose segment
    bases may miss exact optimality by a rounding-sized violation, include/dsp_lp.h): at a midpoint where the segment's basis does not
    verify, the prediction is compared with the exact optimum of the LP there instead.  Returns (segments checked, of them those whose
    basis verified) when exact_bases is False, else the number of segments checked."""
    cnt, st = int(walk["count"]), int(walk["status"])
    th, ob, d1, d2 = walk["theta"][:cnt], walk["obj"][:cnt], walk["dobj"][:cnt], walk["d2obj"][:cnt]
    assert cnt >= 1 and th[0] == 0.0 and walk["enter"][0] == -1 and walk["leave"][0] == -1, (what, cnt, th[:1])
    assert np.isnan(walk["theta"][cnt:]).all() and (walk["enter"][cnt:] == -1).all(), what
    assert (np.diff(th) >= 0).all(), (what, th)
    bases = replay(t, basis, walk)
    ended = st in (3, 4)                                  # INFEASIBLE / UNBOUNDED: the last event only marks where the curve stops
    if ended:
        assert walk["enter"][cnt - 1] == -1 and walk["leave"][cnt - 1] == -1 and np.isnan(d1[cnt - 1]), what
    last = cnt - 1 if ended else cnt                      # events that open a segment
    p = _p(t, cp, rp, dir_c, dir_r)
    pred = lambda e, x: ob[e] + d1[e] * (x - th[e]) + 0.5 * d2[e] * (x - th[e]) ** 2
    checked = verified = 0
    for e in range(last):
        if e + 1 < cnt:
            end = th[e + 1]
            # continuity: the segment meets the next event's objective
            assert abs(pred(e, end) - ob[e + 1]) <= OBJ_REL * max(1.0, abs(ob[e + 1])), (what, e, pred(e, end), ob[e + 1])
            # the breakpoint: the exact end of this basis' range from th[e]
            c0, r0 = XR.moved(t, cp, rp, dir_c, dir_r, th[e])
            hi = XR.exact_range(t, c0, r0, bases[e], dir_c, dir_r)[1]
            assert abs(th[e] + hi - end) <= THETA_REL * max(1.0, abs(end)), (what, e, th[e], hi, end)
        elif st == 0 and math.isinf(theta_end):
            end = th[e] + 20.0 * p                        # the midpoint is 10 max(1, |p|) past the last event
        elif st == 0:
            end = theta_end
        else:
            continue                                      # MAX_ITER / NUMERICAL: the last segment's end is unknown
        if end > th[e]:
            mid = 0.5 * (th[e] + end)
            c2, r2 = XR.moved(t, cp, rp, dir_c, dir_r, mid)
            if exact_bases:
                obj = float(XR.verify(t, c2, r2, bases[e]))
            else:
                try:
                    obj = float(XR.verify(t, c2, r2, bases[e]))
                    verified += 1
                except E.NotCertified:
                    obj = E.exact_optimum(t, c2, r2 if t.Pr else None).obj
            assert abs(obj - pred(e, mid)) <= OBJ_REL * max(1.0, abs(obj)), (what, e, mid, obj, pred(e, mid))
            checked += 1
    if events:
        for e in range(cnt):
            c2, r2 = XR.moved(t, cp, rp, dir_c, dir_r, th[e])
            try:
                ex = E.exact_optimum(t, c2, r2 if t.Pr else None)
            except E.NotCertified:
                continue                                  # HiGHS' basis at the breakpoint does not repair: no exact optimum to compare
            assert abs(ex.obj - ob[e]) <= OBJ_REL * max(1.0, abs(ex.obj)), (what, e, th[e], ex.obj, ob[e])
    return checked if exact_bases else (checked, verified)


def shape(walk, sign, what=""):
    """slopes of the segments nondecreasing (sign = 1: a pure rparam direction, the objective is convex) or nonincreasing (sign = -1:
    a pure cparam direction, concave), up to rounding"""
    cnt = int(walk["count"]) - (1 if int(walk["status"]) in (3, 4) else 0)
    d1 = walk["dobj"][:cnt]
    if cnt > 1:
        tol = 1e-9 * max(1.0, float(np.abs(d1).max()))
        assert (sign * np.diff(d1) >= -tol).all(), (what, d1)


def pair(out, k, q):
    """the fields of pair (LP k, direction q) of a walk batch"""
    return {f: out[f][k, q] for f in FIELDS}


def breakpoints(walk):
    """the distinct breakpoints of a walk: the thetas where a segment of positive length starts, after event 0"""
    cnt = int(walk["count"]) - (1 if int(walk["status"]) in (3, 4) else 0)
    th = walk["theta"][:cnt]
    last = np.r_[th[1:] != th[:-1], True]                   # the last event of each run at equal theta defines the segment
    return th[last], np.flatnonzero(last)


def curve(walk, p):
    """(value, slope) of a walk's curve at theta values p (up to its last event when it did not end OPTIMAL)"""
    cnt = int(walk["count"]) - (1 if int(walk["status"]) in (3, 4) else 0)
    th = walk["theta"][:cnt]
    e = np.clip(np.searchsorted(th, p, side="right") - 1, 0, cnt - 1)
    d = p - th[e]
    return walk["obj"][e] + walk["dobj"][e] * d + 0.5 * walk["d2obj"][e] * d * d, walk["dobj"][e] + walk["d2obj"][e] * d


def against_mirror(walk, mirror, what=""):
    """one walk against oracle/parametric_numpy.walk of the same pair: the same status; the same log (event count, theta to
    THETA_REL, obj / dobj / d2obj to OBJ_REL, NaNs in the same places) -> 'same'.  Where a near tie between the two arithmetics sends
    the degenerate pivots at a breakpoint different ways the logs differ (other zero-length events, or a segment split where the slope
    does not change), but the curves must not: at every event of either log and every midpoint between them, the same value and slope
    to OBJ_REL -> 'tie'"""
    assert int(walk["status"]) == int(mirror["status"]), (what, walk["status"], mirror["status"])
    near = lambda a, b, rel: np.array_equal(np.isnan(a), np.isnan(b)) and bool(
        (np.abs(a - b)[~np.isnan(b)] <= rel * np.maximum(1.0, np.abs(b[~np.isnan(b)]))).all())
    c = int(walk["count"])
    if int(mirror["count"]) == c and all(near(walk[f][:c], mirror[f][:c], THETA_REL if f == "theta" else OBJ_REL)
                                         for f in ("theta", "obj", "dobj", "d2obj")):
        return "same"
    end = lambda w: w["theta"][int(w["count"]) - 1]
    assert abs(end(walk) - end(mirror)) <= THETA_REL * max(1.0, abs(end(mirror))) or int(walk["status"]) == 0, (what, end(walk), end(mirror))
    pts = np.unique(np.concatenate([walk["theta"][:c], mirror["theta"][:int(mirror["count"])]]))
    pts = pts[np.r_[True, np.diff(pts) > THETA_REL * np.maximum(1.0, np.abs(pts[1:]))]]     # one point per breakpoint of both
    if int(walk["status"]) != 0:
        pts = pts[pts <= min(end(walk), end(mirror))]
    pts = np.concatenate([pts, 0.5 * (pts[1:] + pts[:-1]), pts[-1:] + max(1.0, abs(pts[-1]))])
    tol = THETA_REL * np.maximum(1.0, np.abs(pts))
    pts = pts[(np.abs(pts[:, None] - np.concatenate([walk["theta"][:c], mirror["theta"][:int(mirror["count"])]])[None]) > tol[:, None]).all(1)
              | (pts == 0.0)]                                # values away from the breakpoints (within rounding of one, either side is right)
    if int(walk["status"]) != 0:
        pts = pts[pts <= min(end(walk), end(mirror))]
    (va, sa), (vb, sb) = curve(walk, pts), curve(mirror, pts)
    assert near(va, vb, OBJ_REL), (what, pts[np.argmax(np.abs(va - vb))], np.abs(va - vb).max())
    assert near(sa, sb, OBJ_REL), (what, "slope", pts[np.argmax(np.abs(sa - sb))])
    return "tie"
