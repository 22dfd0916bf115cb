"""TEST INFRASTRUCTURE: builds tests/emu/emu_crossover.cpp (the host structure builders and the CTA body of
dispatches_b200/csrc/dsp_crossover.cuh compiled with g++ on the lock-step SIMT emulator, one warp standing for the CTA) and calls it
through ctypes."""
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
LIB = HERE / "libemu_crossover.so"
_lib = None

# the paths of xo::lp_body that XO_TRACE counts, in the order of dsp_crossover.cuh's TR_* events: push pivots and push reinversions;
# cleanup primal pivots (degenerate ones also counted apart), bound flips, dual pivots, iterations under Bland's rule and reinversions;
# artificials pivoted out, redundant rows met (an artificial that stays basic, once per round) and cleanup rounds
TRACE = ("push_pivot", "push_reinvert", "primal_pivot", "primal_degenerate", "bound_flip", "dual_pivot", "bland", "cleanup_reinvert",
         "artificial_out", "redundant_row", "round")


def build(force=False):
    deps = [HERE / "emu_crossover.cpp", HERE / "simt_emu.h", ROOT / "dispatches_b200" / "csrc" / "dsp_crossover.cuh",
            ROOT / "dispatches_b200" / "csrc" / "dsp_sens.cuh"]
    if force or not LIB.exists() or any(d.stat().st_mtime > LIB.stat().st_mtime for d in deps):
        cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", str(LIB),
               str(HERE / "emu_crossover.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ failed:\n" + r.stderr[-3000:])
    return LIB


def run(t, cparams, rparams, status, x, y, max_pivots=0, col_perm=None, row_perm=None):
    """dict(obj, x, y, col_status, row_basic, status, pivots, trace) of the emulated CTA body, x / y / basis in template order;
    trace: {path in TRACE: [N] times each LP took it}"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.emu_crossover.argtypes = [C.c_int] * 5 + [C.c_void_p] * 19 + [C.c_double, C.c_int] + [C.c_void_p] * 3 + \
            [C.c_longlong, C.c_void_p, C.c_void_p, C.c_longlong] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 8
        assert _lib.emu_crossover_trace_events() == len(TRACE)
    I = internal(t, col_perm, row_perm)
    cperm = np.arange(t.n) if I["col_perm"] is None else I["col_perm"]
    rperm = np.arange(t.m) if I["row_perm"] is None else I["row_perm"]
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
                b0=f64(np.asarray(t.b0, float)[rperm]), bmp=i32(I["Bm"].indptr), bmi=i32(I["Bm"].indices), bmv=f64(I["Bm"].data),
                u0=f64(np.asarray(t.u0, float)[cperm[:t.nb]]), ump=i32(I["Um"].indptr), umi=i32(I["Um"].indices), umv=f64(I["Um"].data),
                om=f64(t.omap if t.Pr else np.zeros(1)), ocm=f64(t.ocmap if t.Pc else np.zeros(1)),
                tq=i32(I["q"] if t.amap is not None else [0]), tp=i32(t.amap[2] if t.amap is not None else [0]),
                tc=f64(t.amap[3] if t.amap is not None else [0.0]), st=i32(status))
    out = dict(obj=np.empty(N), x=np.empty((N, t.n)), y=np.empty((N, t.m)), col_status=np.empty((N, t.n), np.int8),
               row_basic=np.empty((N, t.m), np.int8), status=np.empty(N, np.int32), pivots=np.empty(N, np.int32))
    trace = np.zeros((N, len(TRACE)), np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    nt = len(t.amap[0]) if t.amap is not None else 0
    k = keep
    r = _lib.emu_crossover(t.m, t.n, t.nb, t.Pc, t.Pr, vp(k["Ap"]), vp(k["Ai"]), vp(k["Av"]), vp(k["cperm"]), vp(k["rperm"]),
                           vp(k["c0"]), vp(k["cmp"]), vp(k["cmi"]), vp(k["cmv"]), vp(k["b0"]), vp(k["bmp"]), vp(k["bmi"]), vp(k["bmv"]),
                           vp(k["u0"]), vp(k["ump"]), vp(k["umi"]), vp(k["umv"]), vp(k["om"]), vp(k["ocm"]), float(t.o0), nt,
                           vp(k["tq"]), vp(k["tp"]), vp(k["tc"]), N, vp(cp), vp(rp), rstride, vp(k["st"]), vp(x), vp(y), int(max_pivots),
                           vp(out["obj"]), vp(out["x"]), vp(out["y"]), vp(out["col_status"]), vp(out["row_basic"]), vp(out["status"]),
                           vp(out["pivots"]), vp(trace))
    assert r == 0
    out["trace"] = {name: trace[:, q] for q, name in enumerate(TRACE)}
    return out
