"""The dense cluster kernel's algorithm on the CPU: its cluster factorisation and substitutions (csrc/dsp_dense.cuh, cluster_column /
cluster_panel / cluster_fwd / cluster_bwd) on the SIMT emulator with the ranks run one after another between the cluster barriers,
against the single-CTA routines (bit for bit) and numpy, including zero and negative pivots and m not a multiple of the tile; the
ranks' tile ownership; the numpy mirror on the design LP past the old 1024-row limit against its exact optima; and the C ABI's argument checks of
dsp_lp_template_create_dense_cluster, which come before any CUDA call."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import real_lps as R
from dispatches_b200 import solver as S
from oracle import ipm_dense_numpy as ID
from oracle.highs import host_cores

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / "libemu_dense_cluster.so"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", str(so),
                        str(HERE / "emu" / "emu_dense_cluster.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(so))
    lib.emu_dense_cluster_factor_solve.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4
    lib.emu_dense_single_factor_solve.argtypes = [C.c_int] + [C.c_void_p] * 4
    lib.emu_dense_tiles_doubles.restype = C.c_longlong
    return lib


def _run(lib, M, r, csize):
    """(cluster result, single-CTA result) of factor + solve of M padded with unit rows: each (factor tiles, dinv, solution)"""
    m = M.shape[0]
    nt = -(-m // 64)
    mp = nt * 64
    Mp = np.eye(mp); Mp[:m, :m] = M
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    out = []
    for k in range(2):
        v = np.zeros(mp); v[:m] = r
        dinv = np.zeros(mp)
        G = np.zeros(lib.emu_dense_tiles_doubles(nt))
        if k == 0:
            assert lib.emu_dense_cluster_factor_solve(nt, csize, vp(Mp), vp(v), vp(dinv), vp(G)) == 0
        else:
            assert lib.emu_dense_single_factor_solve(nt, vp(Mp), vp(v), vp(dinv), vp(G)) == 0
        out.append((G, dinv, v))
    return out, Mp


# (m, C): ranks with several target tiles per column (m = 300, C = 2), one tile each, and ranks without any (C = 8 > 6 tile rows)
@pytest.mark.parametrize("m,csize", [(130, 2), (300, 2), (300, 4), (380, 8)])
def test_cluster_routines_match_the_single_cta_routines(emu, m, csize):
    rng = np.random.default_rng(m + csize)
    A = rng.normal(size=(m, m + 20)) * (rng.random((m, m + 20)) < 0.3)
    A[np.arange(m), np.arange(m)] += 1.0
    d = np.exp(rng.uniform(0, np.log(1e6), m + 20))
    M = (A * d) @ A.T
    r = rng.normal(size=m)
    (cl, one), Mp = _run(emu, M, r, csize)
    for a, b in zip(cl, one):
        assert np.array_equal(a, b)
    ref = np.linalg.solve(M, r)
    assert np.abs(cl[2][:m] - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max())
    assert not cl[2][m:].any()
    Lm, dm = ID.ldl_blocked(Mp[None])
    assert np.allclose(cl[1], dm[0], rtol=1e-8, atol=0)          # the mirror sums in another order


@pytest.mark.parametrize("m,kind,csize", [(129, "zero", 2), (200, "negative", 4), (250, "zero", 8)])
def test_cluster_routines_pivot_rule(emu, m, kind, csize):
    """a zero row and an indefinite matrix: non-positive pivots get 1/d = 0 as in the single-CTA routines and the mirror"""
    rng = np.random.default_rng(m + 7)
    A = rng.normal(size=(m, m + 10)) * (rng.random((m, m + 10)) < 0.3)
    A[np.arange(m), np.arange(m)] += 1.0
    M = A @ A.T
    dead = [3, m // 2, m - 1]
    if kind == "zero":
        M[dead, :] = 0.0; M[:, dead] = 0.0
    else:
        M = M - np.diag(np.where(np.isin(np.arange(m), dead), 2.0 * np.diag(M), 0.0))
    r = rng.normal(size=m)
    (cl, one), Mp = _run(emu, M, r, csize)
    for a, b in zip(cl, one):
        assert np.array_equal(a, b)
    Lm, dm = ID.ldl_blocked(Mp[None])
    assert (dm[0][:m] == 0).any() and np.array_equal(cl[1] == 0, dm[0] == 0)
    assert np.allclose(cl[1], dm[0], rtol=1e-9, atol=0)
    sol = ID.ldl_solve(Lm, dm, np.r_[r, np.zeros(Mp.shape[0] - m)][None])[0]
    assert np.abs(cl[2] - sol).max() <= 1e-8 * max(1.0, np.abs(sol).max())


@pytest.mark.parametrize("nt", [17, 18, 33, 40, 64])
@pytest.mark.parametrize("csize", [2, 4, 8])
def test_ranks_own_every_target_tile_once(emu, nt, csize):
    """for every block column J the ranks' target tiles (I, J), I >= J (from first_own, every C-th row) are disjoint and cover the column"""
    for J in range(nt):
        seen = []
        for rank in range(csize):
            seen += list(range(emu.emu_dense_first_own(J, rank, csize), nt, csize))
        assert sorted(seen) == list(range(J, nt))


# LPs of the certified design sets the mirror runs: the reference's case and two perturbed ones baked; an exact-zero quarter, an
# all-zero PV series and cf = 1 hours with a PV series per LP
MIRROR_LPS = {False: [0, 1, 2], True: [R.SOLAR_PV.index(c) for c in ("zero_hours", "all_zero", "cf_one")]}


@pytest.mark.parametrize("T", [72, 96])
def test_mirror_solves_the_design_lp_past_1024_rows(T):
    """the numpy mirror of the dense kernels' iteration on the design LP with m = 15 T + 3 > 1024 rows, baked and with a PV series per
    LP, against the certified exact optima (real_lps, the sets the GPU suite runs the cluster kernel on) through check_exact, and
    within 1e-8 of the exact objective.  The mirror at T = 168 (m = 2 523) is not run here: it takes about a minute per LP."""
    procs = host_cores()
    for pv, s in ((False, R.solar_design(T, 8, procs=procs)), (True, R.solar_design_pv(T, 8 if T == 72 else 6, procs=procs))):
        assert 1024 < s.t.m <= 4096 and (s.t.amap is not None) == pv
        q = s.take(np.array(MIRROR_LPS[pv]))
        obj, status, x, y = [], [], [], []
        for k in range(len(q)):
            c, b, u, kk = q.t.instantiate(q.cparams[k], q.rparams[k])
            r = ID.solve_batch(q.t.matrix(q.rparams[k]), b[None], c[None], u[None], rho=q.t.meta.get("reg_primal", 1e-8))
            obj.append(r["obj"][0] + kk); status.append(r["status"][0]); x.append(r["x"][0]); y.append(r["y"][0])
        assert (np.array(status) == ID.OPTIMAL).all(), status
        e = R.check_exact(q, np.array(obj), np.array(status), np.stack(x), np.stack(y), what=(T, pv))
        assert e["obj"] < 1e-8, e
        print(T, "PV series per LP" if pv else "baked", R.fmt(e))


def _desc(m, n, keep):
    """dsp_lp_desc of the LP [I I] x = 1 with u = 1 (m rows, n = 2m columns)"""
    A_ptr = np.arange(0, 2 * m + 1, 2, dtype=np.int32)
    A_idx = np.stack([np.arange(m), m + np.arange(m)], 1).ravel().astype(np.int32)
    keep.update(A_ptr=A_ptr, A_idx=A_idx, A_val=np.ones(2 * m), b0=np.ones(m), u0=np.ones(n), c0=np.ones(n),
                zp_n=np.zeros(n + 1, np.int32), zp_m=np.zeros(m + 1, np.int32), zi=np.zeros(1, np.int32), zv=np.zeros(1))
    p = lambda k: keep[k].ctypes.data_as(C.c_void_p)
    e_n = S._ParamMap(p("zp_n"), p("zi"), p("zv"))
    e_m = S._ParamMap(p("zp_m"), p("zi"), p("zv"))
    return S._LpDesc(m=m, n=n, Pc=0, Pr=2, A_ptr=p("A_ptr"), A_idx=p("A_idx"), A_val=p("A_val"), c0=p("c0"), cmap=e_n, b0=p("b0"),
                     bmap=e_m, u0=p("u0"), umap=e_n, o0=0.0, omap=None, ocmap=None)


def test_abi_argument_checks(cuda_solver_lib):
    lib = cuda_solver_lib
    assert hasattr(lib, "dsp_lp_template_create_dense_cluster") and "dsp_lp_template_create_dense_cluster" in S.EXPORTS
    h = C.c_void_p()
    keep = {}
    d = _desc(4097, 2 * 4097, keep)
    assert lib.dsp_lp_template_create_dense_cluster(C.byref(d), 0, None, None, None, None, C.byref(h)) == -1
    assert b"m <= 4096" in lib.dsp_lp_last_error()
    d = _desc(8, 16, keep)
    i32 = lambda *v: np.array(v, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    coef = np.ones(1)
    row, col, par = i32(0), i32(1), i32(0)                 # (0, 1) is not in the pattern of [I I]
    assert lib.dsp_lp_template_create_dense_cluster(C.byref(d), 1, vp(row), vp(col), vp(par), vp(coef), C.byref(h)) == -1
    assert b"not in the sparsity pattern" in lib.dsp_lp_last_error()
    row, col, par = i32(0), i32(0), i32(5)                 # rparams index 5 >= Pr
    assert lib.dsp_lp_template_create_dense_cluster(C.byref(d), 1, vp(row), vp(col), vp(par), vp(coef), C.byref(h)) == -1
    assert b"index out of range" in lib.dsp_lp_last_error()
    assert b"dsp_lp_template_create_dense_cluster" in lib.dsp_lp_last_error()


C_SNIPPET = r"""
#include <stdio.h>
#include <string.h>
#include "dsp_lp.h"
int main(void) {
    enum { M = 4097 };
    static int32_t ptr[M + 1], idx[M], zp[M + 1], zi[1];
    static double val[M], u0[M], zv[1];
    for (int i = 0; i < M; ++i) { ptr[i + 1] = i + 1; idx[i] = i; val[i] = 1.0; u0[i] = 1.0; }
    dsp_param_map e = {zp, zi, zv};
    dsp_lp_desc d = {M, M, 0, 0, ptr, idx, val, NULL, e, NULL, e, u0, e, 0.0, NULL, NULL};
    dsp_template *t = NULL;
    int rc = dsp_lp_template_create_dense_cluster(&d, 0, NULL, NULL, NULL, NULL, &t);
    printf("%d %s\n", rc, dsp_lp_last_error());
    return rc == DSP_E_ARG && t == NULL && strstr(dsp_lp_last_error(), "m <= 4096") ? 0 : 1;
}
"""


def test_c_program_calls_the_new_entry_point(tmp_path):
    from dispatches_b200.csrc import build
    lib = build.build()
    src = tmp_path / "cluster.c"
    src.write_text(C_SNIPPET)
    exe = tmp_path / "cluster"
    r = subprocess.run([shutil.which("gcc") or "gcc", "-std=c99", "-O1", "-Wall", f"-I{ROOT / 'include'}", str(src), f"-L{lib.parent}",
                        "-ldsp_lp", f"-Wl,-rpath,{lib.parent}", "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
