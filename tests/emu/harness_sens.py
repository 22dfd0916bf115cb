"""TEST INFRASTRUCTURE: builds tests/emu/emu_sens.cpp (the host structure builder and the warp body of
dispatches_b200/csrc/dsp_sens.cuh compiled with g++ on the lock-step SIMT emulator) and calls it through ctypes."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import scipy.sparse as sp

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
LIB = HERE / "libemu_sens.so"
_lib = None


def build(force=False):
    deps = [HERE / "emu_sens.cpp", HERE / "simt_emu.h", ROOT / "dispatches_b200" / "csrc" / "dsp_sens.cuh"]
    if force or not LIB.exists() or any(d.stat().st_mtime > LIB.stat().st_mtime for d in deps):
        cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", str(LIB), str(HERE / "emu_sens.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ failed:\n" + r.stderr[-3000:])
    return LIB


def internal(t, col_perm=None, row_perm=None):
    """the template in an internal order: internal column k is template column col_perm[k] (the bounded ones first), internal row k
    template row row_perm[k]; the arrays dsp_lp.cu keeps on the host, matrix terms as CSR positions of the internal matrix"""
    n, m, nb = t.n, t.m, t.nb
    cperm = np.arange(n) if col_perm is None else np.asarray(col_perm)
    rperm = np.arange(m) if row_perm is None else np.asarray(row_perm)
    assert np.isfinite(t.u0[cperm[:nb]]).all(), "internal order: bounded columns first"
    A = sp.csr_matrix(t.A)[rperm][:, cperm].tocsr()
    A.sort_indices()
    cpos = np.argsort(cperm); rpos = np.argsort(rperm)
    Cm = sp.csr_matrix(t.Cmap)[cperm].tocsr(); Bm = sp.csr_matrix(t.Bmap)[rperm].tocsr(); Um = sp.csr_matrix(t.Umap)[cperm[:nb]].tocsr()
    q = []
    if t.amap is not None:
        for r, c in zip(t.amap[0], t.amap[1]):
            i, j = rpos[r], cpos[c]
            row = A.indices[A.indptr[i]:A.indptr[i + 1]]
            hit = np.flatnonzero(row == j)
            assert hit.size == 1, "matrix term outside the pattern of A"
            q.append(A.indptr[i] + hit[0])
    return dict(A=A, Cm=Cm, Bm=Bm, Um=Um, c0=np.asarray(t.c0, float)[cperm], col_perm=None if col_perm is None else cperm,
                row_perm=None if row_perm is None else rperm, q=np.asarray(q, np.int32))


def run(t, cparams, rparams, status, x, y, col_perm=None, row_perm=None, want=(True, True, True)):
    """(rc, d_cparams, d_rparams) of the emulated warp body, in template order (the order of x and y); None where not wanted"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.emu_sens.argtypes = [C.c_int] * 5 + [C.c_void_p] * 17 + [C.c_int] + [C.c_void_p] * 3 + [C.c_longlong, C.c_void_p, C.c_void_p,
                                                                                                        C.c_longlong] + [C.c_void_p] * 6
    I = internal(t, col_perm, row_perm)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    x = f64(x); y = f64(y)
    N = x.shape[0]
    cp = f64(np.asarray(cparams, float).reshape(N, t.Pc)) if t.Pc else None
    rp = f64(rparams) if t.Pr else None
    rstride = 0 if rp is None or rp.ndim == 1 else t.Pr
    keep = dict(Ap=i32(I["A"].indptr), Ai=i32(I["A"].indices), Av=f64(I["A"].data),
                cperm=None if I["col_perm"] is None else i32(I["col_perm"]), rperm=None if I["row_perm"] is None else i32(I["row_perm"]),
                c0=f64(I["c0"]), cmp=i32(I["Cm"].indptr), cmi=i32(I["Cm"].indices), cmv=f64(I["Cm"].data),
                bmp=i32(I["Bm"].indptr), bmi=i32(I["Bm"].indices), bmv=f64(I["Bm"].data),
                ump=i32(I["Um"].indptr), umi=i32(I["Um"].indices), umv=f64(I["Um"].data),
                om=f64(t.omap if t.Pr else np.zeros(1)), ocm=f64(t.ocmap if t.Pc else np.zeros(1)),
                tq=i32(I["q"] if t.amap is not None else [0]), tp=i32(t.amap[2] if t.amap is not None else [0]),
                tc=f64(t.amap[3] if t.amap is not None else [0.0]), st=i32(status))
    rc = np.empty((N, t.n)) if want[0] else None
    dcp = np.empty((N, t.Pc)) if want[1] and t.Pc else None
    drp = np.empty((N, t.Pr)) if want[2] and t.Pr else None
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    nt = len(t.amap[0]) if t.amap is not None else 0
    r = _lib.emu_sens(t.m, t.n, t.nb, t.Pc, t.Pr, vp(keep["Ap"]), vp(keep["Ai"]), vp(keep["Av"]), vp(keep["cperm"]), vp(keep["rperm"]),
                      vp(keep["c0"]), vp(keep["cmp"]), vp(keep["cmi"]), vp(keep["cmv"]), vp(keep["bmp"]), vp(keep["bmi"]), vp(keep["bmv"]),
                      vp(keep["ump"]), vp(keep["umi"]), vp(keep["umv"]), vp(keep["om"]), vp(keep["ocm"]), nt, vp(keep["tq"]),
                      vp(keep["tp"]), vp(keep["tc"]), N, vp(cp), vp(rp), rstride, vp(keep["st"]), vp(x), vp(y), vp(rc), vp(dcp), vp(drp))
    assert r == 0
    if want[1] and not t.Pc:
        dcp = np.zeros((N, 0))
    if want[2] and not t.Pr:
        drp = np.zeros((N, 0))
    return rc, dcp, drp
