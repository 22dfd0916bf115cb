"""CPU tests of the parametric walk (dsp_lp_parametric): the CTA body of dispatches_b200/csrc/dsp_parametric.cuh on the SIMT emulator, from
exactly verified optimal bases of real, degenerate dispatch LPs, along LMP, size and hydrogen-price directions; against exact arithmetic
(parametric_check), against the ranging of the same basis, and on small LPs built to end INFEASIBLE, UNBOUNDED or MAX_ITER."""
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import lp_template as LT, scenarios as SC, templates as TP  # noqa: E402
import exact_lp as E  # noqa: E402
import exact_ranging as XR  # noqa: E402
import parametric_check as PC  # noqa: E402
import real_lps as R  # noqa: E402

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

T = 24
EXACT_SAMPLE = 2          # LPs per set whose walks go through the exact checks


def _wind_dirs(t, rp, hours=(0, 11, 19), pem=False):
    """LMP hours (1 $/MWh), then wind (1 MW: wind_kw cf_t of the LP's own capacity factors and wind_kw), battery (1 MW)(, the hydrogen
    price (1 $/kg) and the PEM size (1 MW)), and one direction moving an LMP and the battery size together -> (dir_c, dir_r, sign)
    with sign 1 / -1 for a pure rparam / cparam direction (convex / concave) and 0 for the mixed one"""
    rows_c, rows_r, sign = [], [], []
    add = lambda c, r, s_: (rows_c.append(c), rows_r.append(r), sign.append(s_))
    for h in hours:
        c = np.zeros(t.Pc); c[h] = 1.0
        add(c, np.zeros(t.Pr), -1)
    r = np.zeros(t.Pr); r[:T] = 1e3 * rp[:T] / rp[T + 1]; r[T + 1] = 1e3
    add(np.zeros(t.Pc), r, 1)
    r = np.zeros(t.Pr); r[T] = 1e3
    add(np.zeros(t.Pc), r, 1)
    if pem:
        c = np.zeros(t.Pc); c[T] = 1.0
        add(c, np.zeros(t.Pr), -1)
        r = np.zeros(t.Pr); r[T + 2] = 1e3
        add(np.zeros(t.Pc), r, 1)
    c = np.zeros(t.Pc); c[7] = 1.0
    r = np.zeros(t.Pr); r[T] = 1e2
    add(c, r, 0)
    return np.array(rows_c), np.array(rows_r), np.array(sign)


def _axes(t, n=4):
    """a sample of the cparam axes (every LMP-like parameter of the operation templates) -> (dir_c, dir_r, sign)"""
    q = np.unique(np.linspace(0, t.Pc - 1, min(n, t.Pc)).astype(int))
    dc = np.zeros((len(q), t.Pc)); dc[np.arange(len(q)), q] = 1.0
    return dc, np.zeros((len(q), t.Pr)), -np.ones(len(q), int)


SETS = {
    "c2": lambda: (lambda s: (s,) + _wind_dirs(s.t, s.rparams[0]))(R.c2(4)),
    "c2_battery_from_0": lambda: (lambda s: (s,) + _wind_dirs(s.t, s.rparams[0], hours=(5,)))(
        R._wb(T, SC.c2()[0][[0, 2500, 5000]], SC.c2()[1], SC.c2()[2], 0.0)),
    "nuclear": lambda: (lambda s: (s,) + _axes(s.t))(R.nuclear(T, N=4)),
    "bidder": lambda: (lambda s: (s,) + _axes(s.t))(R.operation("wind_battery_bidder_da", N=4)),
    "wind_battery_pem": lambda: (lambda s: (s,) + _wind_dirs(s.t, s.rparams[0], hours=(3, 18), pem=True))(R.wind_battery_pem(N=4)),
}

_cache = {}


def _walks(name, S=256):
    if (name, S) not in _cache:
        import harness_parametric as HP
        s, dc, dr, sign = SETS[name]()
        N = len(s)
        out = HP.run(s.t, s.cparams, s.rparams, np.zeros(N, np.int32), s.col, s.row_basic, dc, dr if s.t.Pr else None, S=S)
        _cache[(name, S)] = (s, dc, dr, sign, out)
    return _cache[(name, S)]


@needs_gxx
@pytest.mark.parametrize("name", sorted(SETS))
def test_emulated_walks_are_exact(name):
    s, dc, dr, sign, out = _walks(name)
    assert (out["status"] == 0).all(), (name, out["status"])
    checked = 0
    for k in range(EXACT_SAMPLE):
        basis = (s.col[k], s.row_basic[k])
        XR.verify(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, basis)
        for q in range(len(dc)):
            w = PC.pair(out, k, q)
            checked += PC.check_walk(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, basis, w, dc[q], dr[q] if s.t.Pr else None,
                                     events=q < 2, what=(name, k, q))
            if sign[q]:
                PC.shape(w, sign[q], (name, k, q))
            else:
                assert (w["d2obj"][:w["count"]] != 0).any(), (name, k, q)        # c and b move together: piecewise quadratic
    ev = out["count"][:EXACT_SAMPLE]
    print(name, "segments checked exactly", checked, "events per walk mean", ev.mean(), "max", ev.max())
    assert checked >= len(dc) * EXACT_SAMPLE


@needs_gxx
def test_battery_walk_from_zero_flips_fixed_columns_at_the_wrong_bound():
    """at batt_mw = 0 the battery columns are fixed at 0, and a basis may have them at either bound.  Started from a basis with every
    nonbasic battery column at the bound its reduced cost does not ask for, the walk first flips them, zero-length events at theta = 0,
    and then follows the same exact curve"""
    import harness_parametric as HP
    s, dc, dr, sign, out = _walks("c2_battery_from_0")
    q = int(np.flatnonzero((dr[:, T] != 0) & (dc == 0).all(1))[0])
    flips = 0
    for k in range(EXACT_SAMPLE):
        u = s.u[k]
        wrong = (u == 0) & (s.col[k] != 1) & (np.abs(s.r[k]) > 1e-6 * s.csc[k])
        assert wrong.any()
        col = np.where(wrong, 2 - s.col[k], s.col[k]).astype(np.int8)
        basis = (col, s.row_basic[k])
        XR.verify(s.t, s.cparams[k], s.rparams[k], basis)                    # optimal at theta = 0: those columns are fixed
        w = PC.pair(HP.run(s.t, s.cparams[[k]], s.rparams[[k]], np.zeros(1, np.int32), col[None], s.row_basic[[k]], dc[[q]], dr[[q]],
                           S=256), 0, 0)
        c = w["count"]
        zero = (w["theta"][1:c] == 0.0) & (w["enter"][1:c] == -1) & (w["leave"][1:c] >= 0)
        assert set(w["leave"][1:c][zero]) == set(np.flatnonzero(wrong)), (k, w["leave"][:c])
        flips += int(zero.sum())
        assert w["status"] == 0
        PC.check_walk(s.t, s.cparams[k], s.rparams[k], basis, w, dc[q], dr[q], events=False, what=("flipped", k))
        ref = PC.pair(out, k, q)                                               # the same curve as from the unflipped basis
        pts = np.concatenate([w["theta"][:c], ref["theta"][:ref["count"]]])
        pts = np.concatenate([pts, pts + 1.0])
        assert np.allclose(value(w, pts), value(ref, pts), rtol=1e-9, atol=1e-9 * abs(ref["obj"][0]))
    assert flips >= 1


def value(w, p):
    """the walk's curve at theta values p"""
    c = int(w["count"]) - (1 if int(w["status"]) in (3, 4) else 0)
    th = w["theta"][:c]
    e = np.searchsorted(th, p, side="right") - 1
    d = p - th[e]
    return w["obj"][e] + w["dobj"][e] * d + 0.5 * w["d2obj"][e] * d * d


@needs_gxx
@pytest.mark.parametrize("name", ["c2", "nuclear", "wind_battery_pem"])
def test_first_segment_is_the_ranging_bit_for_bit(name):
    import harness_ranging as H
    s, dc, dr, sign, out = _walks(name)
    g = H.run(s.t, s.cparams, s.rparams, np.zeros(len(s), np.int32), s.col, s.row_basic, dc, dr if s.t.Pr else None)
    assert np.array_equal(out["dobj"][:, :, 0], g["dobj"]) and np.array_equal(out["d2obj"][:, :, 0], g["d2obj"])
    more = out["count"] > 1
    assert np.array_equal(out["theta"][:, :, 1][more], g["hi"][more])
    assert np.isinf(g["hi"][~more]).all()


@needs_gxx
def test_max_iter_keeps_the_log_and_batch_position():
    import harness_parametric as HP
    s, dc, dr, sign, full = _walks("c2")
    S = 3
    out = HP.run(s.t, s.cparams, s.rparams, np.zeros(len(s), np.int32), s.col, s.row_basic, dc, dr, S=S)
    long_ = full["count"] > S
    assert long_.any()
    assert (out["status"][long_] == 1).all() and (out["count"][long_] == S).all()
    assert (out["status"][~long_] == full["status"][~long_]).all()
    for f in PC.FIELDS[:7]:
        assert np.array_equal(out[f], full[f][:, :, :S], equal_nan=True), f
    k = np.array([2, 0, 2, 3])                                        # the same pairs elsewhere in the batch, and per-LP directions
    per = HP.run(s.t, s.cparams[k], s.rparams[k], np.zeros(4, np.int32), s.col[k], s.row_basic[k],
                 np.broadcast_to(dc, (4,) + dc.shape), np.broadcast_to(dr, (4,) + dr.shape), S=256)
    for f in PC.FIELDS:
        assert np.array_equal(per[f], full[f][k], equal_nan=True), f


@needs_gxx
def test_theta_end_and_non_optimal_inputs():
    import harness_parametric as HP
    s, dc, dr, sign, full = _walks("c2")
    N, K = len(s), len(dc)
    te = np.full(K, 50.0)
    out = HP.run(s.t, s.cparams, s.rparams, np.array([0, 1, 2, 3], np.int32), s.col, s.row_basic, dc, dr, theta_end=te, S=256)
    assert list(out["status"][:, 0]) == [0, 1, 2, 3] and (out["count"][1:] == 0).all()
    assert np.isnan(out["theta"][1:]).all() and (out["enter"][1:] == -1).all() and (out["leave_to"][1:] == -1).all()
    for q in range(K):
        c, cf = out["count"][0, q], full["count"][0, q]
        inside = full["theta"][0, q, :cf] < 50.0
        assert c == inside.sum() and out["status"][0, q] == 0
        assert np.array_equal(out["theta"][0, q, :c], full["theta"][0, q, :c])


@needs_gxx
@pytest.mark.parametrize("case", ["free_wind", "solar_design_pv"])
def test_directions_that_move_A_are_nan(case):
    import harness_parametric as HP
    if case == "free_wind":
        N = 2
        lmp, cf, _, _ = SC.c2(N)
        t = TP.wind_battery_design_free_wind(T, None, 10000.0)
        rp = np.ascontiguousarray(np.broadcast_to(np.asarray(cf, float)[..., :T], (N, T)) - TP.CF_NOMINAL)
        s = R.certify(t, lmp, rp)
    else:
        s = R.solar_design_pv(24)
    t = s.t
    in_A = np.zeros(t.Pr, bool)
    in_A[np.asarray(t.amap[2], int)] = True
    q = int(np.flatnonzero(in_A)[0])
    dr = np.zeros((2, t.Pr)); dr[1, q] = 1.0
    dc = np.zeros((2, t.Pc)); dc[0, 0] = 1.0
    out = HP.run(t, s.cparams, s.rparams, np.zeros(len(s), np.int32), s.col, s.row_basic, dc, dr, S=8)
    assert (out["status"][:, 1] == 2).all() and (out["count"][:, 1] == 0).all() and np.isnan(out["theta"][:, 1]).all()
    assert (out["count"][:, 0] >= 1).all() and np.isin(out["status"][:, 0], (0, 1)).all(), out["status"]   # OPTIMAL or S reached


def _tiny(name, Pc, Pr, build):
    B = LT.TemplateBuilder(name, Pc, Pr)
    build(B)
    return B.build()


def _walk_tiny(t, cp, rp, dc, dr, S=16):
    import harness_parametric as HP
    c, b, u, _ = t.instantiate(cp, rp)
    A = t.matrix(rp).tocsc(copy=True)
    A.sort_indices()
    col, rb = E.exact_optimum(t, cp, rp if t.Pr else None).basis
    out = HP.run(t, cp[None], rp[None] if t.Pr else None, np.zeros(1, np.int32), col[None], rb[None], dc[None] if dc is not None else None,
                 dr[None] if dr is not None else None, S=S)
    return (col, rb), PC.pair(out, 0, 0)


@needs_gxx
def test_infeasible_unbounded_endings():
    # min x  s.t.  x + y = b, 0 <= x, y <= 1, from b = 1.5 upwards: x reaches 1 at b = 2 and no column can take its place
    t = _tiny("two_boxes", 1, 1, lambda B: (lambda x, y: (B.cost(x, (0.0, {0: 1.0})), B.eq("r", {x: 1.0, y: 1.0}, (0.0, {0: 1.0}))))(
        B.var("x", ub=1.0), B.var("y", ub=1.0)))
    basis, w = _walk_tiny(t, np.array([1.0]), np.array([1.5]), np.zeros(1), np.ones(1))
    assert w["status"] == 3 and w["count"] == 2 and w["theta"][1] == 0.5 and w["enter"][1] == -1 and np.isnan(w["dobj"][1])
    PC.check_walk(t, np.array([1.0]), np.array([1.5]), basis, w, np.zeros(1), np.ones(1), what="two_boxes")
    # min -x  s.t.  x + s = 5, x <= u: x sits at u = 2; moving u down, it reaches 0 at theta = 2 and then no point is feasible
    t = _tiny("shrinking_bound", 0, 1, lambda B: (lambda x, s_: (B.cost(x, (-1.0, {})), B.eq("r", {x: 1.0, s_: 1.0}, 5.0)))(
        B.var("x", ub=(0.0, {0: 1.0})), B.var("s")))
    basis, w = _walk_tiny(t, np.zeros(0), np.array([2.0]), None, -np.ones(1))
    assert w["status"] == 3 and w["count"] == 2 and w["theta"][1] == 2.0 and w["obj"][1] == 0.0
    PC.check_walk(t, np.zeros(0), np.array([2.0]), basis, w, None, -np.ones(1), what="shrinking_bound")
    # min c x  s.t.  x - z = 1, z >= 0 without an upper bound: c moves from 2 down through 0, where the LP becomes unbounded
    t = _tiny("ray", 1, 0, lambda B: (lambda x, z: (B.cost(x, (0.0, {0: 1.0})), B.eq("r", {x: 1.0, z: -1.0}, 1.0)))(
        B.var("x"), B.var("z")))
    basis, w = _walk_tiny(t, np.array([2.0]), np.zeros(0), -np.ones(1), None)
    assert w["status"] == 4 and w["count"] == 2 and w["theta"][1] == 2.0 and w["obj"][1] == 0.0, w
    PC.check_walk(t, np.array([2.0]), np.zeros(0), basis, w, -np.ones(1), None, what="ray")


@needs_gxx
@pytest.mark.parametrize("case", ["battery", "pem"])
def test_size_curve_minimum_is_the_exact_design_optimum(case):
    """walked from 0, the minimum of the battery-size curve of templates.wind_battery is the exact optimum of templates.wind_battery_design
    (the PEM-size curve of wind_battery_pem without a battery: of its design_opt="PEM" template)"""
    import harness_parametric as HP
    N = 4
    lmp, cf, W, _ = SC.c2(N, seed=11 if case == "battery" else 5)
    cf = np.broadcast_to(np.asarray(cf, float)[..., :T], (N, T))
    if case == "battery":
        cp, rp = lmp, TP.wind_battery_rparams(T, cf, W, 0.0)
        t, td, q = TP.wind_battery(T), TP.wind_battery_design(T), T
    else:
        cp, rp = np.concatenate([lmp, np.full((N, 1), 2.5)], axis=1), TP.wind_battery_rparams(T, cf, W, 0.0, pem_mw=0.0)
        t, td, q = TP.wind_battery_pem(T, with_battery=False), TP.wind_battery_pem(T, with_battery=False, pem_design=True), T + 2
    s = R.certify(t, cp, rp)
    dr = np.zeros((1, t.Pr)); dr[0, q] = 1e3
    out = HP.run(t, s.cparams, s.rparams, np.zeros(N, np.int32), s.col, s.row_basic, None, dr, S=512)
    assert (out["status"] == 0).all()
    for k in range(N):
        ex = E.exact_optimum(td, cp[k], rp[k]).obj
        best = out["obj"][k, 0, :out["count"][k, 0]].min()
        assert abs(best - ex) <= 1e-12 * max(1.0, abs(ex)), (case, k, best, ex)


@needs_gxx
def test_curves_value_evaluates_the_piecewise_curve():
    """solver.Curves.value on the emulated walks (CPU tensors) against the segments evaluated one by one, NaN past the stop of an
    INFEASIBLE walk"""
    torch = pytest.importorskip("torch")
    from dispatches_b200 import solver as S
    s, dc, dr, sign, out = _walks("c2")
    cv = S.Curves(*(torch.as_tensor(out[f]) for f in PC.FIELDS))
    p = np.array([0.0, 3.0, 50.0, 500.0, 5000.0])
    got = cv.value(torch.as_tensor(p)).numpy()
    want = np.array([[value(PC.pair(out, k, q), p) for q in range(len(dc))] for k in range(len(s))])
    assert np.array_equal(got, want)
    w = dict(theta=np.array([0.0, 0.5, np.nan]), obj=np.array([1.0, 1.5, np.nan]), dobj=np.array([1.0, np.nan, np.nan]),
             d2obj=np.array([0.0, np.nan, np.nan]), enter=np.array([-1, -1, -1], np.int32), leave=np.array([-1, -1, -1], np.int32),
             leave_to=np.array([-1, -1, -1], np.int8), count=np.array(2, np.int32), status=np.array(3, np.int32))
    one = S.Curves(*(torch.as_tensor(w[f])[None, None] for f in PC.FIELDS))
    assert np.allclose(one.value(torch.tensor([0.25, 0.5]))[0, 0].numpy(), [1.25, 1.5])
    assert torch.isnan(one.value(torch.tensor([0.75]))).all()
    w.update(theta=np.array([0.0, 0.5]), obj=np.array([1.0, 1.5]), dobj=np.array([1.0, 2.0]), d2obj=np.zeros(2),
             enter=np.array([-1, 3], np.int32), leave=np.array([-1, 4], np.int32), leave_to=np.array([-1, 0], np.int8),
             status=np.array(1, np.int32))                    # MAX_ITER: nothing is known past the last event
    one = S.Curves(*(torch.as_tensor(w[f])[None, None] for f in PC.FIELDS))
    v = one.value(torch.tensor([0.25, 0.5, 0.75]))[0, 0].numpy()
    assert np.allclose(v[:2], [1.25, 1.5]) and np.isnan(v[2])
    w["status"] = np.array(0, np.int32)                          # OPTIMAL up to theta_end
    one = S.Curves(*(torch.as_tensor(w[f])[None, None] for f in PC.FIELDS), theta_end=torch.tensor([[1.0]], dtype=torch.float64))
    v = one.value(torch.tensor([0.75, 1.0, 1.25]))[0, 0].numpy()
    assert np.allclose(v[:2], [2.0, 2.5]) and np.isnan(v[2])


# (LP, direction) pairs where a near tie between the kernel's and the mirror's arithmetic sends degenerate pivots different ways: the
# logs differ, the curves agree (parametric_check.against_mirror)
TIES = {"bidder": [(0, 1), (0, 2)], "c2": [(1, 3), (2, 3), (2, 4), (2, 5)], "c2_battery_from_0": [(0, 2), (0, 3), (2, 2), (2, 3)],
        "nuclear": [],
        "wind_battery_pem": [(0, 0), (0, 5), (0, 6), (1, 4), (1, 6), (2, 0), (2, 2), (2, 5), (2, 6), (3, 1), (3, 5), (3, 6)]}


@needs_gxx
@pytest.mark.parametrize("name", sorted(SETS))
def test_emulated_walks_against_the_numpy_mirror(name):
    """every (LP, direction) pair of the set against oracle/parametric_numpy.py, which factorises every basis from scratch with LU
    solves: the same status and log, or, at the pinned near ties, the same curve"""
    from oracle import parametric_numpy as PN
    s, dc, dr, sign, out = _walks(name)
    ties = []
    for k in range(len(s)):
        for q in range(len(dc)):
            m = PN.walk(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, s.col[k], s.row_basic[k], dc[q], dr[q] if s.t.Pr else None)
            if PC.against_mirror(PC.pair(out, k, q), m, what=(name, k, q)) == "tie":
                ties.append((k, q))
    print(name, "near ties", ties, "of", out["count"].size, "pairs")
    assert ties == TIES[name], (name, ties)
