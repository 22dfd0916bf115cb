"""TEST INFRASTRUCTURE: builds tests/emu/emu_parametric.cpp (the CTA body of dispatches_b200/csrc/dsp_parametric.cuh compiled with g++ on
the lock-step SIMT emulator, one warp standing for the CTA) and calls it through ctypes."""
from __future__ import annotations

import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
if str(HERE) not in sys.path:
    sys.path.insert(0, str(HERE))
from harness_sens import internal  # noqa: E402

ROOT = HERE.parent.parent
LIB = HERE / "libemu_parametric.so"
_lib = None

FIELDS = ("theta", "obj", "dobj", "d2obj", "enter", "leave", "leave_to", "count", "status")


def build(force=False):
    deps = [HERE / "emu_parametric.cpp", HERE / "simt_emu.h", ROOT / "dispatches_b200" / "csrc" / "dsp_parametric.cuh",
            ROOT / "dispatches_b200" / "csrc" / "dsp_ranging.cuh", ROOT / "dispatches_b200" / "csrc" / "dsp_crossover.cuh",
            ROOT / "dispatches_b200" / "csrc" / "dsp_sens.cuh"]
    if force or not LIB.exists() or any(d.stat().st_mtime > LIB.stat().st_mtime for d in deps):
        cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", str(LIB),
               str(HERE / "emu_parametric.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ failed:\n" + r.stderr[-3000:])
    return LIB


def run(t, cparams, rparams, status, col_status, row_basic, dir_c, dir_r, theta_end=np.inf, S=64):
    """dict(theta, obj, dobj, d2obj, enter, leave, leave_to [N,K,S], count, status [N,K]) of the emulated walks from the bases
    (col_status [N,n], row_basic [N,m], template order).  dir_c [K,Pc] / dir_r [K,Pr] shared by the batch, or [N,K,Pc] / [N,K,Pr] per
    LP (either may be None); theta_end a scalar, [K], or [N,K] with per-LP directions."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.emu_parametric.argtypes = [C.c_int] * 5 + [C.c_void_p] * 19 + [C.c_double, C.c_int] + [C.c_void_p] * 3 + \
            [C.c_longlong, C.c_void_p, C.c_void_p, C.c_longlong] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 2 + [C.c_int] + \
            [C.c_void_p, C.c_int] + [C.c_void_p] * 9
    I = internal(t, None, None)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    col_status = np.ascontiguousarray(col_status, np.int8)
    row_basic = np.ascontiguousarray(row_basic, np.int8)
    N = col_status.shape[0]
    K = (dir_c if dir_c is not None else dir_r).shape[-2]
    dc = f64(dir_c) if dir_c is not None and t.Pc else None
    dr = f64(dir_r) if dir_r is not None and t.Pr else None
    per_lp = int(any(d is not None and np.ndim(d) == 3 for d in (dir_c, dir_r)))
    te = f64(np.broadcast_to(np.asarray(theta_end, float), (N, K) if per_lp else (K,)))
    cp = f64(np.asarray(cparams, float).reshape(N, t.Pc)) if t.Pc else None
    rp = f64(rparams) if t.Pr else None
    rstride = 0 if rp is None or rp.ndim == 1 else t.Pr
    keep = dict(Ap=i32(I["A"].indptr), Ai=i32(I["A"].indices), Av=f64(I["A"].data),
                c0=f64(I["c0"]), cmp=i32(I["Cm"].indptr), cmi=i32(I["Cm"].indices), cmv=f64(I["Cm"].data),
                b0=f64(np.asarray(t.b0, float)), bmp=i32(I["Bm"].indptr), bmi=i32(I["Bm"].indices), bmv=f64(I["Bm"].data),
                u0=f64(np.asarray(t.u0, float)[:t.nb]), ump=i32(I["Um"].indptr), umi=i32(I["Um"].indices), umv=f64(I["Um"].data),
                om=f64(t.omap if t.Pr else np.zeros(1)), ocm=f64(t.ocmap if t.Pc else np.zeros(1)),
                tq=i32(I["q"] if t.amap is not None else [0]), tp=i32(t.amap[2] if t.amap is not None else [0]),
                tc=f64(t.amap[3] if t.amap is not None else [0.0]), st=i32(status))
    out = dict(theta=np.empty((N, K, S)), obj=np.empty((N, K, S)), dobj=np.empty((N, K, S)), d2obj=np.empty((N, K, S)),
               enter=np.empty((N, K, S), np.int32), leave=np.empty((N, K, S), np.int32), leave_to=np.empty((N, K, S), np.int8),
               count=np.empty((N, K), np.int32), status=np.empty((N, K), np.int32))
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    nt = len(t.amap[0]) if t.amap is not None else 0
    k = keep
    r = _lib.emu_parametric(t.m, t.n, t.nb, t.Pc, t.Pr, vp(k["Ap"]), vp(k["Ai"]), vp(k["Av"]), None, None,
                            vp(k["c0"]), vp(k["cmp"]), vp(k["cmi"]), vp(k["cmv"]), vp(k["b0"]), vp(k["bmp"]), vp(k["bmi"]), vp(k["bmv"]),
                            vp(k["u0"]), vp(k["ump"]), vp(k["umi"]), vp(k["umv"]), vp(k["om"]), vp(k["ocm"]), float(t.o0), nt,
                            vp(k["tq"]), vp(k["tp"]), vp(k["tc"]), N, vp(cp), vp(rp), rstride, vp(k["st"]), vp(col_status),
                            vp(row_basic), int(K), vp(dc), vp(dr), per_lp, vp(te), int(S), *(vp(out[f]) for f in FIELDS))
    assert r == 0
    return out
