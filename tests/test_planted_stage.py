"""Exact references for the stage kernels, on the CPU: the exact-optimum solver and KKT measure (tests/exact_lp.py), the planted
wind + battery and storage-chain generators (tests/planted_stage.py), and the CUDA sources of stage 2, the long-horizon kernel
and the chain kernel on the lock-step SIMT emulator (tests/emu) against the exact x, y and objective."""
import importlib.util
import pathlib
import shutil

import numpy as np
import pytest

from dispatches_b200 import lp_template as LT
from exact_lp import exact_optimum, kkt_residuals
from oracle import highs as H, lp_models as L
from planted_stage import CHAIN_T, check, planted_chain, planted_wb

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


def _harness(name):
    spec = importlib.util.spec_from_file_location("emu_" + name, pathlib.Path(__file__).parent / "emu" / f"{name}.py")
    h = importlib.util.module_from_spec(spec); spec.loader.exec_module(h)
    h.build()
    return h


@pytest.fixture(scope="module")
def emu():
    return _harness("harness")


@pytest.fixture(scope="module")
def emu_chain():
    return _harness("harness_chain1")


def _kkt_max(p, k):
    return max(kkt_residuals(p.t, p.cparams[k], p.rparams[k], p.x[k], p.y[k]).values())


# ---------------------------------------------------------------------------------------------------------------- generators
@pytest.mark.parametrize("T", [2, 5, 13, 24, 33, 96, 129, 200])
def test_planted_wb_is_exact_and_unique(T):
    """20 draws, >= 90 % certified unique in x and y (planted_wb asserts the rate), exact KKT, margins, and the same optimum from
    HiGHS on the reference's own formulation of the LP (oracle.lp_models)"""
    p = planted_wb(T, 20, seed=3)
    assert p.drawn <= 22 and p.x_margin > 1e-2 and p.r_margin > 1e-3, (p.drawn, p.x_margin, p.r_margin)    # (XY_REL)
    for k in range(0, 20, 7):
        assert _kkt_max(p, k) < 1e-15
        lmp, rp = p.cparams[k], p.rparams[k]
        W, P = rp[T + 1], rp[T]
        ref = H.solve(L.wind_battery_raw(lmp, rp[:T] / W, W / 1e3, P / 1e3))[0]
        assert p.obj[k] == pytest.approx(ref, rel=1e-9)


@pytest.mark.parametrize("T", [13, 24, 96, 200])
def test_planted_wb_full_battery_variant(T):
    """the battery fills to capacity in hour 4: the soc_bound row of that hour has a nonzero dual (zero in the base cycle)"""
    p = planted_wb(T, 20, seed=4, soc=True)
    isb = [i for i, nm in enumerate(p.t.row_names) if nm.startswith("soc_bound")]
    assert (p.y[:, p.t.row_names.index("soc_bound[4]")] != 0).all()
    assert (np.count_nonzero(p.y[:, isb], axis=1) == 1).all()
    base = planted_wb(T, 5, seed=4)
    assert not base.y[:, isb].any()
    assert _kkt_max(p, 0) < 1e-15


@pytest.mark.parametrize("bounded", ["mixed", "all", "none"])
@pytest.mark.parametrize("NF", [2, 3])
@pytest.mark.parametrize("T", sorted(set(CHAIN_T.values()) | {2, 3}))
def test_planted_chain_is_exact_and_recognised(T, NF, bounded):
    p = planted_chain(T, NF, seed=5, N=3, bounded=bounded)          # (asserts detect_chain1 finds T and NF)
    d = LT.detect_chain1(p.t)
    assert sorted(d["col_idx"][d["col_idx"] >= 0]) == list(range(p.t.n))
    for k in range(3):
        e = exact_optimum(p.t, p.cparams[k], p.rparams[k])
        assert e.unique_x and e.unique_y
        # dyadic data: the planted optimum is exact, so the exact solve reproduces it bit for bit
        assert np.array_equal(e.x, p.x[k]) and np.array_equal(e.y, p.y[k]) and e.obj == p.obj[k]
        assert _kkt_max(p, k) == 0.0


def test_kkt_residuals_flag_wrong_duals():
    """zero on the exact optimum; a wrong sign, two swapped rows or a dual-infeasible unbounded column show up"""
    p = planted_wb(24, 2, seed=6)
    t, cp, rp, x, y = p.t, p.cparams[0], p.rparams[0], p.x[0], p.y[0]
    assert max(kkt_residuals(t, cp, rp, x, y).values()) < 1e-15
    i = int(np.argmax(np.abs(y)))
    y1 = y.copy(); y1[i] = -y1[i]
    r1 = kkt_residuals(t, cp, rp, x, y1)
    assert max(r1["gap"], r1["dual_inf"]) > 1e-3
    rows = t.meta["stage_wb"]["row_idx"][5]          # soc and wind rows of hour 5 swapped: what a wrong row_idx writes
    y2 = y.copy(); y2[[rows[0], rows[3]]] = y2[[rows[3], rows[0]]]
    r2 = kkt_residuals(t, cp, rp, x, y2)
    assert max(r2["gap"], r2["dual_inf"]) > 1e-3
    # an unbounded column at 0 priced below zero, with the objective kept: only the dual-infeasibility measure sees it
    q = planted_chain(11, 2, seed=7, N=1, bounded="none")
    c, b, u, _ = q.t.instantiate(q.cparams[0], q.rparams[0])
    r = c - q.t.A.T @ q.y[0]
    j = int(np.flatnonzero(r > 0)[0])
    cp3 = q.cparams[0].copy(); cp3[int(q.t.col_names[j][1:])] -= 2 * r[j]
    r3 = kkt_residuals(q.t, cp3, q.rparams[0], q.x[0], q.y[0])
    assert r3["dual_inf"] > 1e-3 and r3["gap"] < 1e-15 and r3["primal"] == 0.0
    # a primal perturbation
    x4 = x.copy(); x4[int(np.argmax(x))] *= 1 + 1e-6
    assert kkt_residuals(t, cp, rp, x4, y)["primal"] > 1e-8


# ---------------------------------------------------------------------------------------------------------------- emulator
@needs_gxx
@pytest.mark.parametrize("T,Lg,soc", [(5, 2, False), (24, 8, False), (24, 8, True), (96, 32, False), (96, 32, True)])
def test_stage2_source_matches_exact_optimum(emu, T, Lg, soc):
    """stage2::warp_body<L, 3> on 2 warps: several LPs per warp, groups refilled from the ticket counter (the full-battery cycle
    needs T >= 9)"""
    p = planted_wb(T, {2: 40, 8: 12, 32: 5}[Lg], seed=8, soc=soc)
    obj, status, iters, x, y = emu.solve(p.t, p.cparams, p.rparams, Lg, 3, warps=2)
    check(p, obj, status, x, y, what=(T, Lg, soc))


@needs_gxx
@pytest.mark.parametrize("soc", [False, True], ids=["cycle", "full"])
def test_long_source_matches_exact_optimum(emu, soc):
    p = planted_wb(97, 3, seed=9, soc=soc)
    obj, status, iters, x, y = emu.solve_long(p.t, p.cparams, p.rparams, warps=2)
    check(p, obj, status, x, y, what=soc)


@needs_gxx
@pytest.mark.parametrize("bounded", ["mixed", "all", "none"])
@pytest.mark.parametrize("NF", [2, 3])
@pytest.mark.parametrize("Lg", [4, 16])
def test_chain_source_matches_exact_optimum(emu_chain, Lg, NF, bounded):
    p = planted_chain(CHAIN_T[Lg], NF, seed=10, N=10, bounded=bounded)
    obj, status, iters, x, y = emu_chain.solve(p.t, LT.detect_chain1(p.t), p.cparams, p.rparams, Lg, 3, warps=2)
    check(p, obj, status, x, y, what=(Lg, NF, bounded))
