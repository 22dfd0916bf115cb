"""The descriptor-driven single-storage-chain stage kernel (dispatches_b200/csrc/dsp_stage_chain1.cuh): structure recognition on
the templates (lp_template.detect_chain1) and the CUDA SOURCE executed on the lock-step SIMT emulator (tests/emu) against the
oracle -- nuclear dispatch (BASELINE config C3) and the report's tank / turbine LP; templates outside the family are refused."""
import importlib.util
import pathlib
import shutil

import numpy as np
import pytest

from dispatches_b200 import lp_template as LT, scenarios as SC, templates as TP
from exact_lp import kkt_residuals
from oracle import highs as H, ipm_numpy as M, lp_models as L
from planted_stage import KKT_DUAL, KKT_GAP, KKT_PRIMAL

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("emu_harness_chain1", pathlib.Path(__file__).parent / "emu" / "harness_chain1.py")
    h = importlib.util.module_from_spec(spec); spec.loader.exec_module(h)
    h.build()
    return h


def rel_err(a, ref):
    return np.abs(a - ref) / np.maximum(1.0, np.abs(ref))


def test_structure_recognition():
    d = LT.detect_chain1(TP.nuclear(48))
    assert d is not None and d["T"] == 48 and d["NF"] == 2            # the last holdup has no successor: it sits in the free state slot
    assert (d["col_idx"][:, 2] >= 0).all() and d["coef_next"][-1] == 0.0 and (d["coef_next"][:-1] != 0).all()
    assert sorted(d["col_idx"][d["col_idx"] >= 0]) == list(range(TP.nuclear(48).n))
    d = LT.detect_chain1(TP.nuclear_report(24))
    assert d is not None and d["NF"] == 3
    # outside the family: two rows per period and two states (wind + battery), a cycle (periodic state of charge), wide rows
    assert LT.detect_chain1(TP.wind_battery(24)) is None
    assert LT.detect_chain1(TP.wind_battery_pem(24)) is None
    assert LT.detect_chain1(TP.fossil_surrogate(24)) is None


@pytest.mark.parametrize("T,Lg", [(48, 16), (20, 8), (7, 4), (96, 32)])
def test_nuclear_dispatch_matches_oracle_and_band_mirror(emu, T, Lg):
    t = TP.nuclear(T)
    d = LT.detect_chain1(t)
    p = SC.pool()["cluster_days"]
    rng = np.random.default_rng(T)
    N = 11
    days = rng.integers(0, len(p) - 4, N)
    lmp = np.stack([np.concatenate([p[k + i] for i in range(4)])[:T] for k in days]) * rng.lognormal(0, 0.25, (N, T))
    obj, status, iters, x, y = emu.solve(t, d, lmp, None, Lg, 3, warps=2)
    assert (status == 0).all()
    ref = np.array([H.solve(L.nuclear_raw(l))[0] for l in lmp])
    assert rel_err(obj, ref).max() < 1e-7
    # the numpy mirror of the band kernel runs the same algorithm (dense solve): same iteration counts
    mir = [M.solve_template(t, lmp[k], np.zeros(0)) for k in range(3)] if hasattr(M, "solve_template") else None
    if mir is not None:
        assert [m_["iters"] for m_ in mir] == list(iters[:3])
    c, b, u, k = t.instantiate(lmp[0], np.zeros(0))
    assert obj[0] == pytest.approx(c @ x[0] + k, rel=1e-9, abs=1e-9)
    kkt = kkt_residuals(t, lmp[0], None, x[0], y[0])
    assert max(kkt["primal"], kkt["bound"]) <= KKT_PRIMAL and kkt["dual_inf"] <= KKT_DUAL and kkt["gap"] <= KKT_GAP, kkt


def test_report_lp_with_tank_and_turbine_batched_rhs(emu):
    T = 48
    t = TP.nuclear_report(T, demand=2000.0)
    d = LT.detect_chain1(t)
    lmp = SC.pool()["nuc_report_lmp_rt"][1000:1000 + T]
    cases = [(0.75, 40.0, 30000.0, 0.0), (2.0, 200.0, 50000.0, 40.0), (1.25, 120.0, 0.0, 25.0), (1.5, 60.0, 8000.0, 10.0), (1.0, 20.0, 1.0, 1.0)]
    cp = np.array([np.r_[lmp, hp] for hp, _, _, _ in cases]); rp = np.array([[pem, tank, turb] for _, pem, tank, turb in cases])
    obj, status, iters, _, _ = emu.solve(t, d, cp, rp, 16, 3)
    assert (status == 0).all()
    ref = np.array([H.solve(L.nuclear_report_raw(lmp, hp, pem, pem_capex=400.0, tank_cap=tank, turbine_cap=turb, demand=2000.0))[0]
                    for hp, pem, tank, turb in cases])
    assert rel_err(obj, ref).max() < 1e-7
    # a negative capacity is an infeasible bound, reported as such next to regular LPs of the same warp
    rp2 = rp.copy(); rp2[2, 1] = -5.0
    obj, status, _, _, _ = emu.solve(t, d, cp, rp2, 16, 3)
    assert status[2] == 3 and np.isnan(obj[2]) and (np.delete(status, 2) == 0).all()
