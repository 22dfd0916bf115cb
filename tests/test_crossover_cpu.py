"""CPU tests of the crossover post-pass (dsp_lp_crossover): the CTA body of dispatches_b200/csrc/dsp_crossover.cuh on the SIMT emulator,
started from the (x, y) of the numpy interior-point mirrors on real, degenerate dispatch LPs, and every basis it returns verified as an
exact optimum in rational arithmetic (exact_lp.exact_optimum with basis=)."""
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200.lp_template import TemplateBuilder  # noqa: E402
import real_lps as R  # noqa: E402
from crossover_check import PINNED, check_vertices, interior_xy  # noqa: E402

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")


def crossover(s, status, x, y, **kw):
    import harness_crossover as H
    return H.run(s.t, s.cparams, s.rparams, status, x, y, **kw)


SETS = {
    "c2": (lambda: R.c2(16), False),
    "edges": (lambda: R.edges(), False),
    "nuclear": (lambda: R.nuclear(24), False),
    "wind_battery_pem": (lambda: R.wind_battery_pem(), False),
    "solar_battery_pem": (lambda: R.solar("battery_pem"), True),
    "design": (lambda: R.design(24), True),
    "solar_design": (lambda: R.solar_design(24), True),
    "solar_design_pv": (lambda: R.solar_design_pv(24), True),
    "fossil": (lambda: R.fossil(), False),
}
SETS.update({f"operation_{name}": ((lambda name=name: R.operation(name)), False) for name in R.OPERATIONS})


@needs_gxx
@pytest.mark.parametrize("name", sorted(SETS))
def test_real_sets_cross_over_to_exact_optima(name):
    make, dense = SETS[name]
    s = make()
    status, x, y = interior_xy(s, dense)
    if name == "edges":
        # the numpy mirror of the band IPM does not converge on the battery-less edge (every battery column fixed at 0): those inputs
        # are not OPTIMAL and pass through
        nb = R.edge_rows("no_battery")
        assert (status[nb] != 0).all() and (status[np.setdiff1d(np.arange(len(s)), nb)] == 0).all()
    else:
        assert (status == 0).all(), status
    v = crossover(s, status, x, y)
    piv = check_vertices(s, v, status, PINNED.get(name), name)
    assert piv.max() <= 10 * (s.t.m + s.t.n)
    bad = status != 0
    assert (v["status"][bad] == status[bad]).all() and np.isnan(v["x"][bad]).all()


@needs_gxx
def test_reproducible_and_independent_of_batch_position():
    s = R.c2(8)
    status, x, y = interior_xy(s)
    a = crossover(s, status, x, y)
    k = np.array([3, 0, 3, 7, 1])
    b = crossover(s.take(k), status[k], x[k], y[k])
    for f in ("obj", "x", "y", "col_status", "row_basic", "status", "pivots"):
        assert np.array_equal(a[f][k], b[f], equal_nan=True), f


def _redundant_row_lp():
    """min c'x over x0 + x1 = 4, x1 + x2 = 3 and their sum x0 + 2 x1 + x2 = 7 (a redundant row), 0 <= x <= 5, c = cparams"""
    B = TemplateBuilder("redundant", 3, 0)
    xs = [B.var(f"x{j}", ub=5.0) for j in range(3)]
    for j in xs:
        B.cost(j, (0.0, {j: 1.0}))
    B.eq("r0", {xs[0]: 1.0, xs[1]: 1.0}, 4.0)
    B.eq("r1", {xs[1]: 1.0, xs[2]: 1.0}, 3.0)
    B.eq("r2", {xs[0]: 1.0, xs[1]: 2.0, xs[2]: 1.0}, 7.0)
    return B.build()


@needs_gxx
def test_redundant_row_keeps_its_artificial_basic_at_zero():
    t = _redundant_row_lp()
    cp = np.array([[1.0, 2.0, 1.0], [1.0, 1.0, 1.0], [0.0, 0.0, 0.0], [-1.0, 3.0, 2.0]])
    s = R.certify(t, cp, None)
    status, x, y = interior_xy(s)
    assert (status == 0).all()
    v = crossover(s, status, x, y)
    assert (v["status"] == 0).all()
    assert (v["row_basic"].sum(1) == 1).all()             # exactly one artificial stays basic: the rows have rank 2
    check_vertices(s, v, status, what="redundant row")
    A = t.A.toarray()
    for k in range(len(cp)):
        assert np.abs(A @ v["x"][k] - t.b0).max() <= 1e-12
        assert (v["y"][k][v["row_basic"][k] == 1] == 0.0).all() or np.abs(v["y"][k][v["row_basic"][k] == 1]).max() <= 1e-15


@needs_gxx
def test_non_optimal_inputs_pass_through():
    s = R.c2(6)
    status, x, y = interior_xy(s)
    status = np.array([0, 1, 2, 3, 0, 1], np.int32)
    v = crossover(s, status, x, y)
    bad = status != 0
    assert (v["status"] == status).sum() >= bad.sum() and (v["status"][bad] == status[bad]).all()
    assert np.isnan(v["x"][bad]).all() and np.isnan(v["y"][bad]).all() and np.isnan(v["obj"][bad]).all()
    assert (v["col_status"][bad] == -1).all() and (v["row_basic"][bad] == -1).all() and (v["pivots"][bad] == 0).all()
    assert (v["status"][~bad] == 0).all() and np.isfinite(v["x"][~bad]).all()


@needs_gxx
def test_pivot_limit_ends_max_iter():
    s = R.operation("wind_battery_bidder_da")
    status, x, y = interior_xy(s)
    full = crossover(s, status, x, y)
    k = int(np.argmax(full["pivots"]))
    assert full["pivots"][k] >= 2
    v = crossover(s.take([k]), status[[k]], x[[k]], y[[k]], max_pivots=1)
    assert v["status"][0] == 1 and v["pivots"][0] <= 1
