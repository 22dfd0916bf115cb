"""The exact reference on real, degenerate dispatch LPs (tests/real_lps.py), on the CPU: the basis certifier against today's
answers on planted LPs, its certification rate on the real sets, a hand-built LP with a known primal and dual optimal face, a
corrupted basis, the exact repair of an infeasible HiGHS basis (planted by hand, and on the PV + battery + hydrogen LPs), and the
CUDA sources of stage 2, the long-horizon kernel and the chain kernel on the lock-step SIMT emulator
(tests/emu) through check_exact."""
import numpy as np
import pytest

import exact_lp as X
import real_lps as R
from dispatches_b200 import lp_template as LT
from dispatches_b200 import templates as TP
from exact_lp import NotCertified, exact_optimum, highs_basis, kkt_residuals
from oracle.highs import host_cores
from planted_stage import XY_REL, planted_chain, planted_wb
from test_planted_stage import _harness, needs_gxx


@pytest.fixture(scope="module")
def emu():
    return _harness("harness")


@pytest.fixture(scope="module")
def emu_chain():
    return _harness("harness_chain1")


def _basis_from_x(e, u):
    """the classification the certifier used before it read HiGHS' basis: strictly inside = basic, else at 0 or at u"""
    fin = np.isfinite(u)
    col = np.where(e.basic, 1, np.where(fin & (e.x == np.where(fin, u, 0.0)) & (e.x > 0), 2, 0)).astype(np.int8)
    return col, np.zeros(len(e.y), bool)


# ---------------------------------------------------------------------------------------------------------------- certifier
@pytest.mark.parametrize("T", [2, 24, 97])
def test_certifier_reproduces_planted_optima(T):
    """on nondegenerate planted LPs HiGHS' basis is the one the strictly-inside classification gives: the same ExactOptimum,
    bit for bit, and every column fixed or inside"""
    p = planted_wb(T, 6, seed=21)
    for k in range(6):
        e = exact_optimum(p.t, p.cparams[k], p.rparams[k])
        u = p.t.instantiate(p.cparams[k], p.rparams[k])[2]
        f = exact_optimum(p.t, p.cparams[k], p.rparams[k], basis=_basis_from_x(e, u))
        for a, b in ((e.x, p.x[k]), (e.y, p.y[k]), (e.x, f.x), (e.y, f.y), (e.r, f.r), (e.basic, f.basic)):
            assert np.array_equal(a, b)
        assert (e.obj, e.lp_mag, e.unique_x, e.unique_y, e.x_margin, e.r_margin) == (p.obj[k], p.lp_mag[k], True, True, f.x_margin, f.r_margin)
        assert (e.fixed == ~e.basic).all() and (e.inside == e.basic).all()


def test_certifier_reproduces_planted_chain_optima():
    p = planted_chain(24, 3, seed=22, N=3)
    for k in range(3):
        e = exact_optimum(p.t, p.cparams[k], p.rparams[k])
        assert np.array_equal(e.x, p.x[k]) and np.array_equal(e.y, p.y[k]) and e.obj == p.obj[k]


@pytest.mark.parametrize("name", ["c2", "c5", "edges", "windows97", "nuclear", "nuclear_report", "fossil"])
def test_real_sets_certify(name):
    """every LP of the sampled real sets certifies (a set raises NotCertified on the first that does not), most are degenerate,
    and the exact optimum satisfies its own KKT conditions and check_exact"""
    s = {"c2": lambda: R.c2(64), "c5": R.c5, "edges": R.edges, "windows97": lambda: R.windows(97, 4), "nuclear": lambda: R.nuclear(48),
         "nuclear_report": lambda: R.nuclear_report(48), "fossil": lambda: R.fossil(168, 4)}[name]()
    assert len(s) == {"c2": 64, "c5": 201, "edges": 4 * len(R.EDGES), "windows97": 4, "nuclear": 16, "nuclear_report": 16, "fossil": 4}[name]
    if name in ("c2", "c5", "edges", "windows97", "fossil"):
        assert not s.unique_y.all()
    e = R.check_exact(s, s.obj, np.zeros(len(s), np.int32), s.x, s.y, what=name)
    assert max(e["primal"], e["bound"]) < 1e-14
    assert (s.pivots == 0).all()


EXISTING = {"c2": lambda: R.c2(64), "c5": R.c5, "edges": R.edges, "windows33": lambda: R.windows(33), "nuclear": lambda: R.nuclear(48),
            "nuclear_report": lambda: R.nuclear_report(48), "fossil": lambda: R.fossil(168, 4), "design": R.design,
            "pem": lambda: R.wind_battery_pem(24, True), **{o: (lambda o=o: R.operation(o)) for o in R.OPERATIONS}}


@pytest.mark.parametrize("name", sorted(EXISTING))
def test_existing_sets_need_no_repair(name):
    """HiGHS' basis verifies as it is on the sets that certified before the repair existed: no pivot, and on a sample of each set
    the same ExactOptimum, bit for bit, as the verification of that basis without any repair (an explicit ``basis=``)"""
    s = EXISTING[name]()
    assert (s.pivots == 0).all()
    for k in np.linspace(0, len(s) - 1, 3).astype(int):
        e = exact_optimum(s.t, s.cparams[k], s.rparams[k])
        c, b, u, _ = s.t.instantiate(s.cparams[k], s.rparams[k])
        A = s.t.matrix(s.rparams[k]).tocsc(copy=True)
        A.sort_indices()
        f = exact_optimum(s.t, s.cparams[k], s.rparams[k], basis=highs_basis(c, A, b, u))
        assert e.pivots == f.pivots == 0
        for a, g in ((e.x, s.x[k]), (e.y, s.y[k]), (e.r, s.r[k]), (e.x, f.x), (e.y, f.y), (e.r, f.r), (e.basic, f.basic),
                     (e.fixed, f.fixed), (e.inside, f.inside)):
            assert np.array_equal(a, g)
        assert (e.obj, e.lp_mag, e.unique_x, e.unique_y, e.x_margin, e.r_margin) == (f.obj, f.lp_mag, f.unique_x, f.unique_y,
                                                                                      f.x_margin, f.r_margin)


SOLAR = {**{f"solar_{z}": (lambda z=z: R.solar(z)) for z in R.SOLAR_SIZES}, "solar_design24": lambda: R.solar_design(24),
         "solar_design48": lambda: R.solar_design(48), "solar_design_pv24": lambda: R.solar_design_pv(24),
         "solar_design_pv48": lambda: R.solar_design_pv(48)}


@pytest.mark.parametrize("name", sorted(SOLAR))
def test_solar_sets_certify(name):
    """the PV + battery + hydrogen LPs certify only through the repair: HiGHS drops the 1.2e-16 entry of sin(pi) or leaves row slacks
    and basic columns 1e-14 .. 1e-11 outside their bounds in exact arithmetic.  They are degenerate in x and y."""
    s = SOLAR[name]()
    assert len(s) == 8 and s.pivots.max() > 0 and s.pivots.max() <= X.max_pivots(s.t.m)
    assert not s.unique_x.any() and not s.unique_y.any()
    e = R.check_exact(s, s.obj, np.zeros(len(s), np.int32), s.x, s.y, what=name)
    assert max(e["primal"], e["bound"]) < 1e-13              # x* rounded to binary64: holdups of 1e6 mol next to flows of 1e-2
    if name.startswith("solar_design") and "_pv" not in name:
        assert 0.0 < np.abs(s.t.A.data).min() < 1e-15                # the sin(pi) hour, as the kernels receive it


# the repair's pivots, LP by LP, on the 96-hour design LPs (m = 1 443): the baked set needs up to 95, past the 64 that used to be the
# limit for every LP.  The counts are pinned so that a change of the repair's rules shows.
LONG_DESIGN = {"solar_design96": (lambda: R.solar_design(96, 8, procs=host_cores()), [95, 58, 77, 81, 65, 70, 73, 45]),
               "solar_design_pv96": (lambda: R.solar_design_pv(96, 6, procs=host_cores()), [49, 0, 0, 0, 8, 4])}


@pytest.mark.parametrize("name", sorted(LONG_DESIGN))
def test_long_design_sets_certify(name):
    """the 96-hour design LPs certify through the repair, within its limit, and the repaired basis given back through basis= verifies
    as it is, to the same optimum bit for bit (the week-long LPs, about 70 s each on one core, certify in the GPU suite)"""
    make, pivots = LONG_DESIGN[name]
    s = make()
    assert s.t.m == 1443 and s.pivots.tolist() == pivots and s.pivots.max() < X.max_pivots(s.t.m)
    assert not s.unique_x.any() and not s.unique_y.any()
    e = R.check_exact(s, s.obj, np.zeros(len(s), np.int32), s.x, s.y, what=name)
    assert max(e["primal"], e["bound"]) < 1e-13
    k = int(np.argmax(s.pivots))
    f = exact_optimum(s.t, s.cparams[k], s.rparams[k], basis=(s.col[k], s.row_basic[k]))
    assert f.pivots == 0
    for a, g in ((f.x, s.x[k]), (f.y, s.y[k]), (f.r, s.r[k]), (f.fixed, s.fixed[k]), (f.inside, s.inside[k]),
                 (f.basis[0], s.col[k]), (f.basis[1], s.row_basic[k])):
        assert np.array_equal(a, g)
    assert f.obj == s.obj[k]


@pytest.mark.parametrize("T", [24, 48])
def test_solar_pv_series_have_their_cases(T):
    """the per-LP series hold exact zero hours, an all-zero series, cf = 1 hours and a perturbed reserve; the dyadic LP is the baked
    template's LP, and its exact optimum is the baked one's bit for bit"""
    lmp, load, cfs, reserve = R.solar_pv_series(T, 8)
    case = {c: i for i, c in enumerate(R.SOLAR_PV)}
    assert (cfs[case["zero_hours"]] == 0).sum() >= T // 4 and (cfs[case["all_zero"]] == 0).all() and (cfs[case["cf_one"]] == 1).any()
    assert (reserve[case["reserve"]] != 100.0).all() and (reserve[np.arange(8) != case["reserve"]] == 100.0).all()
    assert np.array_equal(cfs[case["reference"]], np.tile(R._solar_reference()[1]["pv_cfs"], T // 24))
    s = R.solar_design_pv(T)
    k = case["dyadic"]
    tb = TP.solar_battery_hydrogen_design(T, cfs[k])
    e = exact_optimum(tb, lmp[k], load[k] * 1e3)
    assert np.array_equal(e.x, s.x[k]) and np.array_equal(e.y, s.y[k]) and e.obj == s.obj[k]


def test_reference_tank_without_battery_is_infeasible_in_exact_arithmetic():
    """the reference sizes the tank for exactly its 100 MW reserve: in binary64 that tank backs 8.6e-14 kW less, and with no battery
    the night-time reserve rows cannot be met.  The repair proves it (its ratio test finds no entering column), which is why
    real_lps.solar sizes that tank 1 % larger."""
    lmp0, d = R._solar_reference()
    with pytest.raises(NotCertified, match="infeasible in exact arithmetic"):
        exact_optimum(TP.solar_battery_hydrogen(24), lmp0, TP.solar_rparams(24, d["pv_cfs"], 200.0, d["load_mw"])[0])


def _cover_lp(b, surplus):
    """min x1 + 2 x2  s.t.  x1 + x2 - s = b (surplus: a column s >= 0) or x1 + x2 = b, x >= 0.  Optimum x1 = b, y = 1."""
    B = LT.TemplateBuilder("cover", Pc=1, Pr=0)
    x1, x2 = B.var("x1"), B.var("x2")
    B.cost(x1, 1.0); B.cost(x2, 2.0)
    row = {x1: 1.0, x2: 1.0}
    if surplus:
        row[B.var("s")] = -1.0
    B.eq("r", row, b)
    return B.build()


@pytest.mark.parametrize("surplus", [True, False], ids=["basic_column", "basic_row_slack"])
def test_repair_of_a_planted_basis(monkeypatch, surplus):
    """HiGHS' basis replaced by a dual feasible one that is 1e-9 primal infeasible -- the surplus column basic at -b, or the row's
    slack basic at b -- is repaired in one pivot to the exact optimum x1 = b, y = 1.  Given explicitly, the same basis raises; 1e-7
    off, it is too far to repair."""
    t = _cover_lp(1e-9, surplus)
    col = np.zeros(t.n, np.int8)
    if surplus:
        col[t.col_names.index("s")] = 1
    planted = (col, np.array([not surplus]))
    monkeypatch.setattr(X, "highs_basis", lambda *a: planted)
    e = exact_optimum(t, np.zeros(1), None)
    assert e.pivots == 1 and e.x[t.col_names.index("x1")] == 1e-9 and e.x[t.col_names.index("x2")] == 0.0
    assert e.y[0] == 1.0 and e.obj == 1e-9 and e.basic[t.col_names.index("x1")]
    with pytest.raises(NotCertified):
        exact_optimum(t, np.zeros(1), None, basis=planted)
    with pytest.raises(NotCertified, match="too far to repair"):
        exact_optimum(_cover_lp(1e-7, surplus), np.zeros(1), None)


def test_repair_refuses_a_dual_infeasible_basis(monkeypatch):
    """min x1 + 2 x2 - x3  s.t.  x1 + x2 = 1e-9,  x3 + x4 = 1: the basis {row slack 0, x4} is 1e-9 primal infeasible and dual
    infeasible (x3 at 0 with r = -1) -- the repair does not start"""
    B = LT.TemplateBuilder("two_rows", Pc=1, Pr=0)
    v = [B.var(f"x{j}") for j in range(1, 5)]
    B.cost(v[0], 1.0); B.cost(v[1], 2.0); B.cost(v[2], -1.0)
    B.eq("r0", {v[0]: 1.0, v[1]: 1.0}, 1e-9)
    B.eq("r1", {v[2]: 1.0, v[3]: 1.0}, 1.0)
    t = B.build()
    col = np.zeros(t.n, np.int8)
    col[t.col_names.index("x4")] = 1
    rb = np.array([n == "r0" for n in t.row_names])
    monkeypatch.setattr(X, "highs_basis", lambda *a: (col, rb))
    with pytest.raises(NotCertified, match="primal and dual infeasible"):
        exact_optimum(t, np.zeros(1), None)
    monkeypatch.undo()
    e = exact_optimum(t, np.zeros(1), None)
    assert e.obj == -1.0 + 1e-9 and e.pivots == 0


def test_edge_set_has_its_edges():
    s = R.edges()
    z = R.edge_rows("zero_prices")
    assert (s.cparams[z] == 0).all() and (s.lp_mag[z] == 0).all() and (s.csc[z] == 0).all()
    assert (s.cparams[R.edge_rows("negative_prices")] < 0).any(1).all()
    assert (s.cparams[R.edge_rows("spike")] == 10000.0).any(1).all()
    assert (s.cparams[R.edge_rows("whole_dollars")] == np.round(s.cparams[R.edge_rows("whole_dollars")])).all()
    assert ((s.rparams[R.edge_rows("zero_cf"), :24] == 0).sum(1) >= 3).all()
    nb = R.edge_rows("no_battery")
    assert (s.u[nb][np.isfinite(s.u[nb])] == 0).all()
    # c = 0: the gap and dual measures are not applicable; the primal ones still measure
    k = kkt_residuals(s.t, s.cparams[z[0]], s.rparams[z[0]], s.x[z[0]], s.y[z[0]] + 1.0)
    assert k["gap"] is None and k["dual_inf"] is None and k["primal"] < 1e-15


def _face_lp():
    """min -x1 - x2 - x4  s.t.  x1 + x2 + x3 = 1,  x4 + x5 = 1,  x4 + x6 = 1,  x >= 0.
    Primal face: x1 + x2 = 1, x3 = 0, x4 = 1, x5 = x6 = 0.  Dual face: y0 = -1, y1 + y2 = -1 with y1, y2 in [-1, 0]."""
    B = LT.TemplateBuilder("face", Pc=1, Pr=0)
    v = [B.var(f"x{j}") for j in range(1, 7)]
    for j in (0, 1, 3):
        B.cost(v[j], -1.0)
    B.eq("r0", {v[0]: 1.0, v[1]: 1.0, v[2]: 1.0}, 1.0)
    B.eq("r1", {v[3]: 1.0, v[4]: 1.0}, 1.0)
    B.eq("r2", {v[3]: 1.0, v[5]: 1.0}, 1.0)
    t = B.build()
    cols = [t.col_names.index(f"x{j}") for j in range(1, 7)]
    rows = [t.row_names.index(f"r{i}") for i in range(3)]
    return t, cols, rows


def test_certifier_on_a_primal_and_dual_degenerate_lp():
    t, c, r = _face_lp()
    s = R.certify(t, np.zeros((1, 1)), None)
    e = exact_optimum(t, np.zeros(1), None)
    x, y = e.x[c], e.y[r]
    assert e.obj == -2.0 and not e.unique_x and not e.unique_y
    assert x[0] + x[1] == 1.0 and x[2] == 0.0 and x[3] == 1.0 and x[4] == x[5] == 0.0
    assert y[0] == -1.0 and y[1] + y[2] == -1.0 and -1.0 <= y[1] <= 0.0
    assert e.fixed[c[2]] and not e.fixed[c[0]] and not e.fixed[c[1]] and not e.fixed[c[3]] and e.inside[c[3]]
    # another point of both faces passes check_exact; off the dual face (y1 + y2 != -1) or off the primal one it fails
    xs, ys = np.zeros((1, t.n)), np.zeros((1, t.m))
    xs[0, c] = [0.25, 0.75, 0.0, 1.0, 0.0, 0.0]; ys[0, r] = [-1.0, -0.5, -0.5]
    R.check_exact(s, np.array([-2.0]), np.zeros(1, np.int32), xs, ys)
    bad = ys.copy(); bad[0, r[0]] = -0.999
    with pytest.raises(AssertionError):
        R.check_exact(s, np.array([-2.0]), np.zeros(1, np.int32), xs, bad)
    bad = xs.copy(); bad[0, c[2]] = 1e-3; bad[0, c[0]] -= 1e-3
    with pytest.raises(AssertionError):
        R.check_exact(s, np.array([-2.0]), np.zeros(1, np.int32), bad, ys)


def test_corrupted_basis_raises():
    """a basic column swapped with a nonbasic one, on a planted LP (unique optimum) and on a degenerate C2 LP"""
    p = planted_wb(24, 1, seed=23)
    c, b, u, _ = p.t.instantiate(p.cparams[0], p.rparams[0])
    col, rb = highs_basis(c, p.t.A.tocsc(), b, u)
    j, k = int(np.flatnonzero(col == 1)[0]), int(np.flatnonzero(col == 0)[0])
    bad = col.copy(); bad[j], bad[k] = 0, 1
    with pytest.raises(NotCertified):
        exact_optimum(p.t, p.cparams[0], p.rparams[0], basis=(bad, rb))
    s = R.c2(64)
    e = exact_optimum(s.t, s.cparams[1], s.rparams[1])
    j = int(np.flatnonzero(e.basic & e.inside)[0]); k = int(np.flatnonzero(e.fixed & (e.x == 0))[0])
    c, b, u, _ = s.t.instantiate(s.cparams[1], s.rparams[1])
    col, rb = highs_basis(c, s.t.A.tocsc(), b, u)
    bad = col.copy(); bad[j], bad[k] = 0, 1
    with pytest.raises(NotCertified):
        exact_optimum(s.t, s.cparams[1], s.rparams[1], basis=(bad, rb))
    bad = col.copy(); bad[k] = 2                      # a column at a bound it does not have, or with the wrong reduced-cost sign
    with pytest.raises(NotCertified):
        exact_optimum(s.t, s.cparams[1], s.rparams[1], basis=(bad, rb))


def test_check_exact_flags_y_moved_along_the_dual_face():
    """swapping the soc and wind duals of one hour keeps y plausible element by element: the inside-column reduced costs see it"""
    s = R.c2(64)
    rows = s.t.meta["stage_wb"]["row_idx"][12]
    y = s.y.copy(); y[:, [rows[0], rows[3]]] = y[:, [rows[3], rows[0]]]
    with pytest.raises(AssertionError):
        R.check_exact(s, s.obj, np.zeros(len(s), np.int32), s.x, y)


# ---------------------------------------------------------------------------------------------------------------- emulator
def _stage_sets():
    return {"c2": R.c2(16, stride=617), "c5": R.c5(16, stride=35041), "edges": R.edges(), "T5": R.windows(5), "T33": R.windows(33),
            "T96": R.windows(96, 4)}


@needs_gxx
@pytest.mark.parametrize("name,Lg", [("T5", 2), ("c2", 8), ("c5", 8), ("edges", 8), ("T33", 16), ("T96", 32)])
def test_stage2_source_on_real_lps(emu, name, Lg):
    """T33 and T96: real windows on which the stage-2 source used to end OPTIMAL with an energy-throughput row off by up to 6e-8
    of the primal scale (the residual test of its two looser branches was relative to 1 + |b| = 2)"""
    s = _stage_sets()[name]
    obj, status, iters, x, y = emu.solve(s.t, s.cparams, s.rparams, Lg, 3, warps=2)
    R.check_exact(s, obj, status, x, y, what=name)


@needs_gxx
def test_long_source_on_real_lps(emu):
    s = R.windows(97, 4)
    obj, status, iters, x, y = emu.solve_long(s.t, s.cparams, s.rparams, warps=2)
    R.check_exact(s, obj, status, x, y)


@needs_gxx
@pytest.mark.parametrize("name,Lg", [("nuclear", 16), ("nuclear_report", 16), ("nuclear24", 8)])
def test_chain_source_on_real_lps(emu_chain, name, Lg):
    s = {"nuclear": lambda: R.nuclear(48, 8), "nuclear_report": lambda: R.nuclear_report(48, 8), "nuclear24": lambda: R.nuclear(24, 8)}[name]()
    d = LT.detect_chain1(s.t)
    assert d["NF"] == (3 if name == "nuclear_report" else 2)
    obj, status, iters, x, y = emu_chain.solve(s.t, d, s.cparams, s.rparams if s.t.Pr else None, Lg, 3, warps=2)
    R.check_exact(s, obj, status, x, y, what=name)
