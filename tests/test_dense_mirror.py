"""The dense kernel's algorithm on the CPU: the numpy mirror (oracle/ipm_dense_numpy.py) on the PV + battery + hydrogen design LP
against HiGHS and the dense-Cholesky mirror, on planted LPs with w > 32 and a fully dense A against their exact optimum, and the CUDA
tile routines of csrc/dsp_dense.cuh (blocked LDL', panel, tensor-core trailing update through its FMA fallback, substitutions) on
the SIMT emulator against numpy -- including zero and negative pivots and sizes that are not a multiple of the tile."""
import ctypes as C
import json
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from dispatches_b200 import templates as TP
from oracle import highs as H, ipm_dense_numpy as ID, ipm_numpy as IN, lp_models as L
from planted_lp import planted, rel

HERE = Path(__file__).resolve().parent
GOLD = json.load(open(HERE / "golden" / "solar_golden.json"))
LMP = np.array(GOLD["lmp_24"])
PAR = dict(pv_mw=0.0, turb_mw=0.0)


def _design_batch(T, N, seed):
    """the reference's case (T = 24) plus perturbed price / load series, as tests/checks/border_mirror_gate.py draws them"""
    d = L.solar_default_series()
    rng = np.random.default_rng(seed)
    lmp0, load0, cfs = np.tile(LMP, T // 24), np.tile(d["load_mw"], T // 24), np.tile(d["pv_cfs"], T // 24)
    lmp = np.vstack([lmp0[None], lmp0[None] * rng.lognormal(0, 0.3, (N - 1, T))])
    load = np.vstack([load0[None], load0[None] * rng.uniform(0.7, 1.2, (N - 1, T))])
    return lmp, load, cfs


@pytest.mark.parametrize("T,N", [(24, 16), (48, 4)])
def test_mirror_solves_the_design_lp(T, N):
    lmp, load, cfs = _design_batch(T, N, 3)
    t = TP.solar_battery_hydrogen_design(T, cfs, **PAR)
    assert t.w > 32 and t.m <= 1024
    X = [t.instantiate(lmp[k], load[k] * 1e3) for k in range(N)]
    b, c, u = (np.array([x[i] for x in X]) for i in (1, 0, 2))
    kc = np.array([x[3] for x in X])
    r = ID.solve_batch(t.A, b, c, u)
    ref = np.array([H.solve(L.solar_battery_hydrogen_raw(lmp[k], True, PAR, pv_cfs=cfs, load_mw=load[k], reserve_mw=np.full(T, 100.0)))[0]
                    for k in range(N)])
    assert (r["status"] == ID.OPTIMAL).all(), r["status"]
    assert (np.abs(r["obj"] + kc - ref) / np.abs(ref)).max() < 1e-8
    if T == 24:
        assert -(r["obj"][0] + kc[0]) * 1e3 == pytest.approx(GOLD["test_solar_batt_hydrogen_optimize"]["expect"]["NPV"]["value"], rel=1e-8)
        dn = IN.solve_batch(t.A.toarray(), b, c, u)         # the dense-Cholesky mirror: the same answers
        assert (dn["status"] == IN.OPTIMAL).all()
        assert np.allclose(r["obj"], dn["obj"], rtol=1e-8, atol=0)


@pytest.mark.parametrize("m,w,full", [(60, 40, False), (90, 64, False), (150, 200, False), (70, 69, True)])
def test_mirror_on_planted_lps(m, w, full):
    p = planted(m, w, seed=4, N=3, full_span=full)
    t = p.t
    assert t.w > 32
    X = [t.instantiate(p.cparams[k], p.rparams[k]) for k in range(3)]
    b, c, u = (np.array([x[i] for x in X]) for i in (1, 0, 2))
    r = ID.solve_batch(t.A, b, c, u)
    assert (r["status"] == ID.OPTIMAL).all()
    obj = r["obj"] + np.array([x[3] for x in X])
    assert (np.abs(obj - p.obj) / np.maximum(1.0, np.abs(p.obj))).max() < 1e-7
    assert rel(r["x"], p.x) < 1e-6 * p.scale and rel(r["y"], p.y) < 1e-6


def test_mirror_infeasible_and_second_attempt():
    p = planted(70, 40, seed=6, N=2)
    X = [p.t.instantiate(p.cparams[k], p.rparams[k]) for k in range(2)]
    b, c, u = (np.array([x[i] for x in X]) for i in (1, 0, 2))
    j = int(np.flatnonzero(np.isfinite(u[1]))[0])
    u[1, j] = -1.0
    r = ID.solve_batch(p.t.A, b, c, u)
    assert r["status"][0] == ID.OPTIMAL
    assert r["status"][1] == ID.INFEASIBLE and np.isnan(r["obj"][1]) and np.isnan(r["x"][1]).all() and r["iters"][1] == 0
    r = ID.solve_batch(p.t.A, b[:1], c[:1], u[:1], max_iter=3)
    assert r["status"][0] != ID.OPTIMAL and r["iters"][0] == 6


# ---------------------------------------------------------------------------------------------------- tile routines on the emulator
@pytest.fixture(scope="module")
def emu():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = HERE / "emu" / "libemu_dense.so"
    root = HERE.parent
    deps = [HERE / "emu" / "emu_dense.cpp", HERE / "emu" / "simt_emu.h", root / "dispatches_b200" / "csrc" / "dsp_dense.cuh",
            root / "dispatches_b200" / "csrc" / "dsp_band.cuh"]
    if not so.exists() or any(d.stat().st_mtime > so.stat().st_mtime for d in deps):
        r = subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", str(so), str(deps[0])],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(so))
    lib.emu_dense_factor_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _run(lib, M, r):
    """the kernel's factor + solve of the m x m matrix M padded with unit rows: (L unit lower, dinv, solution) of the padded system"""
    m = M.shape[0]
    nt = -(-m // ID.TS)
    mp = nt * ID.TS
    Mp = np.eye(mp); Mp[:m, :m] = M
    v = np.zeros(mp); v[:m] = r
    dinv = np.zeros(mp)
    assert lib.emu_dense_factor_solve(nt, Mp.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), dinv.ctypes.data_as(C.c_void_p)) == 0
    Mm = np.eye(mp); Mm[:m, :m] = M
    Lm, dm = ID.ldl_blocked(Mm[None])
    return Mp, dinv, v, Lm[0], dm[0], mp


@pytest.mark.parametrize("m", [63, 64, 65, 129])
def test_tile_routines_match_numpy(emu, m):
    rng = np.random.default_rng(m)
    A = rng.normal(size=(m, m + 20)) * (rng.random((m, m + 20)) < 0.3)
    A[np.arange(m), np.arange(m)] += 1.0
    d = np.exp(rng.uniform(0, np.log(1e6), m + 20))
    M = (A * d) @ A.T
    r = rng.normal(size=m)
    L_, dinv, v, Lm, dm, mp = _run(emu, M, r)
    ref = np.linalg.solve(M, r)
    assert np.abs(v[:m] - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max())
    assert not v[m:].any()
    assert np.allclose(dinv, dm, rtol=1e-10, atol=0) and np.abs(L_ - Lm).max() < 1e-9 * max(1.0, np.abs(Lm).max())


@pytest.mark.parametrize("m,kind", [(65, "zero"), (129, "zero"), (64, "negative"), (130, "negative")])
def test_tile_routines_pivot_rule(emu, m, kind):
    """a zero row (empty row of A) and an indefinite matrix: the non-positive pivots get 1/d = 0, the row is decoupled, and the
    factor is the mirror's"""
    rng = np.random.default_rng(m + 7)
    A = rng.normal(size=(m, m + 10)) * (rng.random((m, m + 10)) < 0.3)
    A[np.arange(m), np.arange(m)] += 1.0
    M = A @ A.T
    dead = [3, m // 2, m - 1]
    if kind == "zero":
        M[dead, :] = 0.0; M[:, dead] = 0.0
    else:
        M = M - np.diag(np.where(np.isin(np.arange(m), dead), 2.0 * np.diag(M), 0.0))      # negative diagonal entries
    r = rng.normal(size=m)
    L_, dinv, v, Lm, dm, mp = _run(emu, M, r)
    assert (dm[:m] == 0).any() and np.array_equal(dinv == 0, dm == 0)
    assert np.allclose(dinv, dm, rtol=1e-9, atol=0)
    assert np.abs(L_ - Lm).max() < 1e-8 * max(1.0, np.abs(Lm).max())
    sol = ID.ldl_solve(Lm[None], dm[None], np.r_[r, np.zeros(mp - m)][None])[0]
    assert np.abs(v - sol).max() <= 1e-8 * max(1.0, np.abs(sol).max())
    if kind == "zero":
        assert (v[dead] == 0).all() and (dinv[dead] == 0).all()
