"""The split band kernel's algebra on the CPU (no GPU): the numpy mirror of its nested-dissection LDL' (oracle/ipm_band_split_numpy.py)
against dense solves, the CUDA source of dispatches_b200/csrc/dsp_band_split.cuh on the SIMT emulator against the mirror, and the
mirror's IPM on real long-horizon templates against HiGHS' certified optima and against the normal-equations mirror oracle/ipm_numpy.py."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from dispatches_b200 import scenarios as SC
from exact_lp import exact_optimum
from dispatches_b200 import templates as TP
from oracle import ipm_band_split_numpy as S
from oracle import ipm_numpy as I

HERE = Path(__file__).resolve().parent / "emu"
ROOT = HERE.parent.parent

# (W, m): the minimum m = 64 W, m not divisible by 32, uneven chunks (m % 32 = 31: 31 chunks one row longer than the last)
CASES = [(1, 64), (1, 95), (2, 128), (2, 161), (4, 256), (4, 287), (8, 512), (8, 543), (8, 700), (16, 1024), (16, 1055), (32, 2048),
         (32, 2079)]


def planted_band(m, W, rng, kind="dominant"):
    """symmetric band matrix of half bandwidth W: diagonally dominant SPD, or an LP-like A D A' (D spanning 1e6)"""
    if kind == "dominant":
        B = np.zeros((m, m))
        for k in range(W + 1):
            B += np.diag(rng.normal(size=m - k), -k)
        M = B + B.T
        return M + np.diag(np.abs(M).sum(1) + 1.0)
    A = np.zeros((m, m + W))
    for i in range(m):
        A[i, i:i + W + 1] = rng.normal(size=W + 1)
    D = np.exp(rng.uniform(0, np.log(1e6), m + W))
    return A @ np.diag(D) @ A.T


@pytest.mark.parametrize("W,m", CASES)
def test_mirror_reproduces_a_dense_solve(W, m):
    rng = np.random.default_rng(10 * W + m)
    M = planted_band(m, W, rng)
    rhs = rng.normal(size=m)
    x = S.band_solve(M, rhs, W)
    ref = np.linalg.solve(M, rhs)
    assert np.abs(x - ref).max() <= 1e-13 * np.abs(ref).max()
    M2 = planted_band(m, W, rng, kind="lp")
    x2 = S.band_solve(M2, rhs, W)
    assert np.abs(M2 @ x2 - rhs).max() <= 1e-9 * np.abs(M2).max() * np.abs(x2).max()


def test_mirror_is_the_ldlt_of_the_permuted_matrix():
    """L D L' of P M P' from the stored factor equals P M P' (the statement the mirror checks)"""
    W, m = 2, 161
    rng = np.random.default_rng(5)
    M = planted_band(m, W, rng)
    F = S.split_factor(S.pack(M, W), W, m)
    cs, r0, _ = S.layout(m)
    inter = [r0[L] + s for L in range(32) for s in range(cs[L] - (W if L < 31 else 0))]
    sep = lambda k: [r0[k] + cs[k] - W + a for a in range(W)]
    order = inter + sum((sep(k) for k in range(15)), []) + sum((sep(k) for k in range(30, 15, -1)), []) + sep(15)
    assert sorted(order) == list(range(m))
    # reconstruct L (unit) and D from solves with unit vectors: x = M^-1 e  ->  compare M^-1 directly
    Minv = np.stack([S.split_solve(F, _split(np.eye(m)[i], m)).reshape(-1)[S.split_index(m)[0]] for i in range(m)], axis=1)
    assert np.abs(Minv @ M - np.eye(m)).max() < 1e-12


def _split(v, m):
    pos, _ = S.split_index(m)
    _, _, Sr = S.layout(m)
    out = np.zeros(Sr * 32)
    out[pos] = v
    return out.reshape(Sr, 32)


def test_zero_and_negative_pivots_give_zero_reciprocals():
    """an all-zero row (interior and separator) and a negative pivot: 1/d = 0, no NaN, the other rows still solved"""
    W, m = 4, 300
    rng = np.random.default_rng(11)
    M = planted_band(m, W, rng)
    cs, r0, _ = S.layout(m)
    dead = [7, r0[3] + cs[3] - 2, r0[15] + cs[15] - 1]          # an interior row, a row of S_3, a row of the middle separator S_15
    for i in dead:
        M[i, :] = 0.0
        M[:, i] = 0.0
    neg = r0[20] + 5
    M[neg, :] = 0.0; M[:, neg] = 0.0; M[neg, neg] = -3.0
    F = S.split_factor(S.pack(M, W), W, m)
    rhs = rng.normal(size=m)
    x = S.split_solve(F, _split(rhs, m)).reshape(-1)[S.split_index(m)[0]]
    assert np.isfinite(x).all()
    keep = np.setdiff1d(np.arange(m), dead + [neg])
    ref = np.linalg.solve(M[np.ix_(keep, keep)], rhs[keep])
    assert np.abs(x[keep] - ref).max() <= 1e-12 * np.abs(ref).max()
    assert (x[dead + [neg]] == 0.0).all()


def test_mirror_refuses_short_chunks():
    with pytest.raises(ValueError):
        S.split_factor(np.zeros((9, 16, 32)), 8, 511)


# ------------------------------------------------------------------------------------------------------------------ emulator
@pytest.fixture(scope="module")
def emu():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = HERE / "libemu_band_split.so"
    deps = [HERE / "emu_band_split.cpp", HERE / "simt_emu.h", ROOT / "dispatches_b200" / "csrc" / "dsp_band_split.cuh"]
    if not so.exists() or any(d.stat().st_mtime > so.stat().st_mtime for d in deps):
        r = subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", str(so),
                            str(HERE / "emu_band_split.cpp")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(str(so))
    L.emu_band_split_factor_solve.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _emu_run(lib, M, rhs, W):
    m = M.shape[0]
    Mb = np.ascontiguousarray(S.pack(M, W))
    _, _, Sr = S.layout(m)
    G = np.zeros((W, Sr, 32))
    v = np.ascontiguousarray(_split(rhs, m))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.emu_band_split_factor_solve(W, m, vp(Mb), vp(G), vp(v)) == 0
    return Mb, G, v


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("W,m", CASES)
def test_emulated_kernel_matches_the_mirror(emu, W, m):
    rng = np.random.default_rng(1000 + 10 * W + m)
    for kind in ("dominant", "lp"):
        M = planted_band(m, W, rng, kind)
        rhs = rng.normal(size=m)
        Mb, G, v = _emu_run(emu, M, rhs, W)
        F = S.split_factor(S.pack(M, W), W, m)
        ref = S.split_solve(F, _split(rhs, m))
        cs, _, Sr = S.layout(m)
        valid = np.arange(Sr)[:, None] < cs[None, :]
        assert _rel(Mb[:, valid], F.Mb[:, valid]) <= 1e-12
        assert _rel(G[:, valid], F.G[:, valid]) <= 1e-12
        assert _rel(v[valid], ref[valid]) <= 1e-12


def test_emulated_kernel_zero_and_negative_pivots(emu):
    W, m = 8, 600
    rng = np.random.default_rng(2)
    M = planted_band(m, W, rng)
    cs, r0, _ = S.layout(m)
    for i in (3, r0[9] + cs[9] - 1, r0[15] + cs[15] - W):
        M[i, :] = 0.0; M[:, i] = 0.0
    M[r0[25] + 2, r0[25] + 2] = -1.0
    rhs = rng.normal(size=m)
    Mb, G, v = _emu_run(emu, M, rhs, W)
    ref = S.split_solve(S.split_factor(S.pack(M, W), W, m), _split(rhs, m))
    assert np.isfinite(v).all()
    valid = np.arange(S.layout(m)[2])[:, None] < cs[None, :]
    assert _rel(v[valid], ref[valid]) <= 1e-12


# ------------------------------------------------------------------------------------------------------------------ IPM mirror
def _lps(name):
    """(template, cparams, rparams) of two real LPs per template"""
    if name.startswith("wind_battery_pem"):
        T = int(name.split("_")[-1])
        p = SC.pool()
        h0 = np.array([1000, 4000])
        idx = h0[:, None] + np.arange(T)[None, :]
        lmp, cf = p["dalmp_303"][idx], p["dacf_303"][idx]
        cp = np.concatenate([lmp, np.full((2, 1), 2.5)], axis=1)
        return TP.wind_battery_pem(T), cp, TP.wind_battery_rparams(T, cf, SC.FIXED_WIND_MW, 150.0, pem_mw=200.0)
    if name == "nuclear_report_672":
        lam = SC.pool()["nuc_report_lmp_rt"]
        cp = np.stack([np.concatenate([lam[h:h + 672], [1.5]]) for h in (100, 3000)])
        return TP.nuclear_report(672), cp, np.array([[120.0, 20000.0, 20.0], [60.0, 5000.0, 10.0]])
    return TP.fossil_surrogate(168), SC.c4(2), np.zeros((2, 0))


@pytest.mark.parametrize("name", ["wind_battery_pem_168", "wind_battery_pem_672", "nuclear_report_672", "fossil_168"])
def test_ipm_mirror_reaches_highs(name):
    t, cps, rps = _lps(name)
    W = S._half_bandwidth(t.w)
    assert t.m >= 64 * W
    its = []
    for cp, rp in zip(cps, rps):
        r = S.solve(t, cp, rp)
        c, b, u, k = t.instantiate(cp, rp)
        ref = exact_optimum(t, cp, rp).obj          # HiGHS' optimal basis, verified in exact arithmetic (tests/exact_lp.py)
        assert r["status"] == S.OPTIMAL
        assert abs(r["obj"] - ref) <= 1e-8 * max(1.0, abs(ref)), (r["obj"], ref)
        g = I.solve_batch(t.A.toarray(), b, c, u) if t.m <= 1000 else None      # dense LAPACK mirror: small m only
        its.append((r["iters"], None if g is None else int(g["iters"][0])))
    print(name, "split mirror / normal-equations mirror iterations:", its)
    for a, b in its:
        if b is not None:
            assert abs(a - b) <= max(5, 0.25 * b)
