"""CPU tests of every path of the crossover's simplex (csrc/dsp_crossover.cuh) on the SIMT emulator: assignment and planted LPs
started where the cleanup has real work (tests/xo_lps.py) -- dual simplex pivots, Bland's rule, bound flips, push pivots,
reinversions, artificials pivoted out and redundant rows, each pinned by a floor on the path counters the emulator build keeps.  Every
OPTIMAL basis verifies as an exact optimum as it is (exact_lp.exact_optimum with basis=), the assignment objectives equal
linear_sum_assignment's bit for bit, the planted LPs return x* and their planted basis, and the NUMERICAL outputs are as
include/dsp_lp.h documents them."""
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

import xo_lps as X  # noqa: E402
from xo_lps import FIELDS, check_basis_exact  # noqa: E402

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

_runs = {}


def emulate(I, **kw):
    import harness_crossover as H
    return H.run(I.t, I.cparams, I.rparams, I.status, I.x, I.y, **kw)


def case(name):
    """(inputs, emulator outputs) of a case of xo_lps.ROWS, run once per session"""
    if name not in _runs:
        I = X.ROWS[name][0]()
        _runs[name] = (I, emulate(I))
    return _runs[name]


@needs_gxx
@pytest.mark.parametrize("name", sorted(X.ROWS))
def test_paths_reach_their_floors(name):
    I, v = case(name)
    _, status, floors = X.ROWS[name]
    assert (v["status"] == status).all(), (name, v["status"])
    got = {path: int(v["trace"][path].sum()) for path in floors}
    assert all(got[p] >= f for p, f in floors.items()), (name, got, floors)
    assert (v["pivots"] <= 10 * (I.t.m + I.t.n)).all()
    print(name, "pivots", v["pivots"].tolist(), {p: a.tolist() for p, a in v["trace"].items() if a.any()})


@needs_gxx
def test_every_path_is_driven_by_some_case():
    import harness_crossover as H
    total = {p: 0 for p in H.TRACE}
    for name in X.ROWS:
        for p, a in case(name)[1]["trace"].items():
            total[p] += int(a.sum())
    assert all(c > 0 for c in total.values()), total


@needs_gxx
@pytest.mark.parametrize("name", sorted(n for n in X.ROWS if X.ROWS[n][1] == 0))
def test_optimal_bases_verify_exactly(name):
    I, v = case(name)
    for k in range(len(I.x)):
        check_basis_exact(I, v, k)


@needs_gxx
@pytest.mark.parametrize("name", sorted(X.ASSIGNMENT_K))
def test_assignment_objective_is_linear_sum_assignment_bit_for_bit(name):
    I, v = case(name)
    k = X.ASSIGNMENT_K[name]
    want = X.assignment_optimum(I.cparams.reshape(-1, k, k))
    assert np.array_equal(v["obj"], want), (name, v["obj"], want)
    assert (v["row_basic"].sum(1) == 1).all()                 # rank 2k - 1: exactly one artificial stays basic, a redundant row
    assert (v["trace"]["redundant_row"] >= 1).all()
    # an integral vertex: a permutation matrix
    assert set(np.unique(v["x"])) <= {0.0, 1.0} and (v["x"].sum(1) == k).all()


@needs_gxx
def test_planted_lps_return_x_star_and_the_planted_basis():
    I, v = case("planted40_at_u")
    p = X.planted40()
    assert (v["status"] == 0).all()
    assert (I.x != p.x).any(1).all()                          # every LP starts away from x*
    for k in range(len(p.x)):
        col, rb = X.planted_basis(p, k)
        assert np.array_equal(v["col_status"][k], col) and np.array_equal(v["row_basic"][k], rb.astype(np.int8)), k
        assert np.abs(v["x"][k] - p.x[k]).max() <= 1e-12 * p.scale, k
        assert np.abs(v["y"][k] - p.y[k]).max() <= 1e-12 * max(1.0, np.abs(p.y[k]).max()), k
        assert abs(v["obj"][k] - p.obj[k]) <= 1e-12 * max(1.0, p.lp_mag[k]), k


@needs_gxx
def test_numerical_outputs_are_as_documented():
    """primal and dual infeasible after the push: DSP_NUMERICAL with the state the crossover stopped in -- finite x / y / obj, a basis
    of m members, and col_status -1 only for a column strictly inside its bounds"""
    I, v = case("planted40_basic_third_zero")
    assert (v["status"] == 2).all()
    assert np.isfinite(v["x"]).all() and np.isfinite(v["y"]).all() and np.isfinite(v["obj"]).all()
    for k in range(len(I.x)):
        _, _, u, _ = I.t.instantiate(I.cparams[k], I.rparams[k])
        cs, x = v["col_status"][k], v["x"][k]
        assert set(np.unique(cs)) <= {-1, 0, 1, 2}
        assert (x[cs == -1] > 0).all() and (x[cs == -1] < u[cs == -1]).all()
        assert (x[cs == 0] == 0).all() and (x[cs == 2] == u[cs == 2]).all()
        assert (cs == 1).sum() + v["row_basic"][k].sum() == I.t.m


@needs_gxx
def test_results_do_not_depend_on_batch_position():
    """the three assignment starts of k = 40 in one permuted batch with repeats, bitwise equal to their own runs"""
    names = ["assign40_zero_cost3", "assign40_identity_cost1000", "assign40_uniform_cost1000"]
    runs = [case(n) for n in names]
    cp = np.concatenate([I.cparams for I, _ in runs]); x = np.concatenate([I.x for I, _ in runs])
    y = np.concatenate([I.y for I, _ in runs]); st = np.concatenate([I.status for I, _ in runs])
    ref = {f: np.concatenate([v[f] for _, v in runs]) for f in FIELDS}
    k = np.random.default_rng(3).permutation(np.resize(np.arange(len(cp)), len(cp) + 4))
    I0 = runs[0][0]
    v = emulate(X.Inputs(I0.t, cp[k], None, st[k], x[k], y[k]))
    for f in FIELDS:
        assert np.array_equal(v[f], ref[f][k], equal_nan=True), f


@needs_gxx
def test_pivot_limit_ends_max_iter_on_an_assignment():
    I, full = case("assign40_zero_cost1000")
    v = emulate(X.Inputs(I.t, I.cparams[:1], None, I.status[:1], I.x[:1], I.y[:1]), max_pivots=1)
    assert full["pivots"][0] > 1 and v["status"][0] == 1 and v["pivots"][0] <= 1
