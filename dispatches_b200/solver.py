"""Python binding of the C-ABI (include/dsp_lp.h) -- ctypes over libdsp_lp.so.

``BatchLPSolver(template)`` is the batched replacement of the reference's per-LP
``pyo.SolverFactory("cbc").solve(m)`` (wind_battery_LMP.py:266-267): the template is uploaded once, then
``solve`` (device tensors in / device tensors out, stream ordered) or ``solve_host`` (numpy in / numpy out,
copies included) handles a whole scenario batch.  torch is used only for device memory and streams.

There is NO CPU fallback: if the CUDA library is missing or no GPU is visible the calls raise.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from pathlib import Path

import numpy as np

from .lp_template import LPTemplate

import os

_LIB_PATH = Path(os.environ.get("DSP_LP_LIB", Path(__file__).resolve().parent / "csrc" / "libdsp_lp.so"))
_lib = None

OPTIMAL, MAX_ITER, NUMERICAL, INFEASIBLE = 0, 1, 2, 3
STATUS_NAMES = {OPTIMAL: "optimal", MAX_ITER: "maxIterations", NUMERICAL: "error", INFEASIBLE: "infeasible"}

KERNEL_AUTO, KERNEL_BAND, KERNEL_STAGE, KERNEL_STAGE_V1, KERNEL_DENSE = 0, 1, 2, 3, 4

EXPORTS = ["dsp_lp_template_create", "dsp_lp_template_set_matrix_params", "dsp_lp_template_set_stage_chain1", "dsp_lp_template_create_csr", "dsp_lp_template_create_dense", "dsp_lp_analyze_csr", "dsp_lp_template_info", "dsp_lp_template_destroy", "dsp_lp_template_set_stage_wb", "dsp_lp_default_opts", "dsp_lp_solve_batch",
           "dsp_lp_solve_batch_host", "dsp_lp_launch_count", "dsp_lp_last_launch", "dsp_lp_last_error",
           "dsp_lp_version", "dsp_lp_fp64_peak_tflops"]


class _ParamMap(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("idx", C.c_void_p), ("val", C.c_void_p)]


class _Desc(C.Structure):
    _fields_ = [("m", C.c_int32), ("n", C.c_int32), ("nb", C.c_int32), ("w", C.c_int32),
                ("Pc", C.c_int32), ("Pr", C.c_int32),
                ("A_ptr", C.c_void_p), ("A_idx", C.c_void_p), ("A_val", C.c_void_p),
                ("asm_ptr", C.c_void_p), ("asm_col", C.c_void_p), ("asm_val", C.c_void_p),
                ("c0", C.c_void_p), ("cmap", _ParamMap),
                ("b0", C.c_void_p), ("bmap", _ParamMap),
                ("u0", C.c_void_p), ("umap", _ParamMap),
                ("o0", C.c_double), ("omap", C.c_void_p), ("ocmap", C.c_void_p)]


class _LpDesc(C.Structure):
    """dsp_lp_desc (include/dsp_lp.h): the plain standard-form LP handed to dsp_lp_template_create_csr"""
    _fields_ = [("m", C.c_int32), ("n", C.c_int32), ("Pc", C.c_int32), ("Pr", C.c_int32),
                ("A_ptr", C.c_void_p), ("A_idx", C.c_void_p), ("A_val", C.c_void_p),
                ("c0", C.c_void_p), ("cmap", _ParamMap),
                ("b0", C.c_void_p), ("bmap", _ParamMap),
                ("u0", C.c_void_p), ("umap", _ParamMap),
                ("o0", C.c_double), ("omap", C.c_void_p), ("ocmap", C.c_void_p)]


class _Opts(C.Structure):
    _fields_ = [("tol", C.c_double), ("feas_tol", C.c_double), ("max_iter", C.c_int32), ("step_frac", C.c_double),
                ("device", C.c_int32), ("reg_primal", C.c_double), ("kernel", C.c_int32)]


class _StageChain1(C.Structure):
    _fields_ = [("T", C.c_int32), ("NF", C.c_int32), ("col_idx", C.c_void_p), ("row_idx", C.c_void_p), ("coef", C.c_void_p),
                ("coef_next", C.c_void_p)]


class _StageWB(C.Structure):
    _fields_ = [("T", C.c_int32), ("a", C.c_double), ("binv", C.c_double), ("half", C.c_double), ("delta", C.c_double),
                ("dur", C.c_double), ("k_rev", C.c_double), ("wcf_off", C.c_int32), ("p_off", C.c_int32),
                ("col_idx", C.c_void_p), ("row_idx", C.c_void_p)]


def load_library():
    """Loads libdsp_lp.so; raises loudly when it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise RuntimeError(f"{_LIB_PATH} is missing: build it with `python -m dispatches_b200.csrc.build` "
                           "(the solver has no CPU fallback)")
    lib = C.CDLL(str(_LIB_PATH))
    lib.dsp_lp_template_create.argtypes = [C.POINTER(_Desc), C.POINTER(C.c_void_p)]
    lib.dsp_lp_template_create.restype = C.c_int
    lib.dsp_lp_template_create_csr.argtypes = [C.POINTER(_LpDesc), C.POINTER(C.c_void_p)]
    lib.dsp_lp_template_create_csr.restype = C.c_int
    lib.dsp_lp_template_create_dense.argtypes = [C.POINTER(_LpDesc), C.POINTER(C.c_void_p)]
    lib.dsp_lp_template_create_dense.restype = C.c_int
    lib.dsp_lp_analyze_csr.argtypes = [C.POINTER(_LpDesc)] + [C.POINTER(C.c_int32)] * 4 + [C.c_void_p, C.c_void_p]
    lib.dsp_lp_analyze_csr.restype = C.c_int
    lib.dsp_lp_template_set_matrix_params.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsp_lp_template_set_matrix_params.restype = C.c_int
    lib.dsp_lp_template_info.argtypes = [C.c_void_p] + [C.POINTER(C.c_int32)] * 4
    lib.dsp_lp_template_info.restype = C.c_int
    lib.dsp_lp_template_destroy.argtypes = [C.c_void_p]
    lib.dsp_lp_template_destroy.restype = None
    lib.dsp_lp_template_set_stage_wb.argtypes = [C.c_void_p, C.POINTER(_StageWB)]
    lib.dsp_lp_template_set_stage_wb.restype = C.c_int
    lib.dsp_lp_template_set_stage_chain1.argtypes = [C.c_void_p, C.POINTER(_StageChain1)]
    lib.dsp_lp_template_set_stage_chain1.restype = C.c_int
    lib.dsp_lp_default_opts.argtypes = [C.POINTER(_Opts)]
    lib.dsp_lp_default_opts.restype = None
    lib.dsp_lp_solve_batch.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(_Opts),
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsp_lp_solve_batch.restype = C.c_int
    lib.dsp_lp_solve_batch_host.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(_Opts),
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dsp_lp_solve_batch_host.restype = C.c_int
    lib.dsp_lp_launch_count.restype = C.c_int64
    lib.dsp_lp_last_launch.argtypes = [C.POINTER(C.c_int32)] * 4
    lib.dsp_lp_last_launch.restype = C.c_int
    lib.dsp_lp_last_error.restype = C.c_char_p
    lib.dsp_lp_version.restype = C.c_char_p
    lib.dsp_lp_fp64_peak_tflops.restype = C.c_double
    _lib = lib
    return lib


def fp64_peak_tflops() -> float:
    """measured FP64 FMA peak of the current device (TFLOP/s)"""
    return float(load_library().dsp_lp_fp64_peak_tflops())


def launch_count() -> int:
    return int(load_library().dsp_lp_launch_count())


def last_launch():
    g, b, s, p = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    load_library().dsp_lp_last_launch(C.byref(g), C.byref(b), C.byref(s), C.byref(p))
    return dict(grid=g.value, block=b.value, smem_bytes=s.value, problems_per_cta=p.value)


@dataclasses.dataclass
class LPResult:
    obj: object          # [N] objective incl. constant (the reference's Objective value, e.g. -NPV*1e-5)
    status: object       # [N] OPTIMAL / MAX_ITER / NUMERICAL
    iters: object        # [N]
    x: object = None     # [N,n] template-space primal (see LPTemplate.col_names / to_model_space)
    y: object = None     # [N,m] row duals


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class BatchLPSolver:
    def __init__(self, template: LPTemplate, tol=1e-9, feas_tol=1e-9, max_iter=60, step_frac=0.9995, kernel=KERNEL_AUTO, reg_primal=None,
                 native_setup=False):
        """native_setup=True hands the library the PLAIN standard-form LP (dsp_lp_template_create_csr): column / row ordering and
        the band assembly list are then derived in C++ (what a C caller or the Pyomo walker uses); the default passes the
        orderings lp_template.finalize() computed (dsp_lp_template_create).  Results are identical up to summation order."""
        self.lib = load_library()
        self.t = template
        t = template
        nb = t.nb
        if t.amap is not None:
            native_setup = True          # per-problem matrix coefficients need the library's own symbolic setup
        # a template whose A A' is wider than the band kernels take runs on the dense kernel: the library gets the plain LP
        self.dense = kernel == KERNEL_DENSE and t.w > 32
        if self.dense:
            if t.amap is not None:
                raise ValueError("the dense kernel does not take per-problem matrix coefficients")
            native_setup = True
        A = t.A.tocsr(); A.sort_indices()
        Cm = t.Cmap.tocsr(); Bm = t.Bmap.tocsr()
        h = C.c_void_p()
        if native_setup:
            Um = t.Umap.tocsr()
            keep = dict(A_ptr=_i32(A.indptr), A_idx=_i32(A.indices), A_val=_f64(A.data),
                        c0=_f64(t.c0), b0=_f64(t.b0), u0=_f64(np.where(np.isfinite(t.u0), t.u0, 1e300)),
                        cm_ptr=_i32(Cm.indptr), cm_idx=_i32(Cm.indices), cm_val=_f64(Cm.data),
                        bm_ptr=_i32(Bm.indptr), bm_idx=_i32(Bm.indices), bm_val=_f64(Bm.data),
                        um_ptr=_i32(Um.indptr), um_idx=_i32(Um.indices), um_val=_f64(Um.data),
                        omap=_f64(t.omap if t.Pr else np.zeros(1)), ocmap=_f64(t.ocmap if t.Pc else np.zeros(1)))
            p = lambda k: keep[k].ctypes.data_as(C.c_void_p)
            d = _LpDesc(m=t.m, n=t.n, Pc=t.Pc, Pr=t.Pr, A_ptr=p("A_ptr"), A_idx=p("A_idx"), A_val=p("A_val"),
                        c0=p("c0"), cmap=_ParamMap(p("cm_ptr"), p("cm_idx"), p("cm_val")),
                        b0=p("b0"), bmap=_ParamMap(p("bm_ptr"), p("bm_idx"), p("bm_val")),
                        u0=p("u0"), umap=_ParamMap(p("um_ptr"), p("um_idx"), p("um_val")),
                        o0=float(t.o0), omap=p("omap"), ocmap=p("ocmap"))
            create = "dsp_lp_template_create_dense" if self.dense else "dsp_lp_template_create_csr"
            rc = getattr(self.lib, create)(C.byref(d), C.byref(h))
            if rc != 0:
                raise RuntimeError(f"{create} failed ({rc}): {self.lib.dsp_lp_last_error().decode()}")
        else:
            Um = t.Umap.tocsr()[:nb]
            keep = dict(A_ptr=_i32(A.indptr), A_idx=_i32(A.indices), A_val=_f64(A.data),
                        asm_ptr=_i32(t.asm_ptr), asm_col=_i32(t.asm_col), asm_val=_f64(t.asm_val),
                        c0=_f64(t.c0), b0=_f64(t.b0), u0=_f64(t.u0[:nb]),
                        cm_ptr=_i32(Cm.indptr), cm_idx=_i32(Cm.indices), cm_val=_f64(Cm.data),
                        bm_ptr=_i32(Bm.indptr), bm_idx=_i32(Bm.indices), bm_val=_f64(Bm.data),
                        um_ptr=_i32(Um.indptr), um_idx=_i32(Um.indices), um_val=_f64(Um.data),
                        omap=_f64(t.omap if t.Pr else np.zeros(1)), ocmap=_f64(t.ocmap if t.Pc else np.zeros(1)))
            p = lambda k: keep[k].ctypes.data_as(C.c_void_p)
            d = _Desc(m=t.m, n=t.n, nb=nb, w=t.w, Pc=t.Pc, Pr=t.Pr,
                      A_ptr=p("A_ptr"), A_idx=p("A_idx"), A_val=p("A_val"),
                      asm_ptr=p("asm_ptr"), asm_col=p("asm_col"), asm_val=p("asm_val"),
                      c0=p("c0"), cmap=_ParamMap(p("cm_ptr"), p("cm_idx"), p("cm_val")),
                      b0=p("b0"), bmap=_ParamMap(p("bm_ptr"), p("bm_idx"), p("bm_val")),
                      u0=p("u0"), umap=_ParamMap(p("um_ptr"), p("um_idx"), p("um_val")),
                      o0=float(t.o0), omap=p("omap"), ocmap=p("ocmap"))
            rc = self.lib.dsp_lp_template_create(C.byref(d), C.byref(h))
            if rc != 0:
                raise RuntimeError(f"dsp_lp_template_create failed ({rc}): {self.lib.dsp_lp_last_error().decode()}")
        self.handle = h
        if t.amap is not None:
            ar, ac, ak, av = _i32(t.amap[0]), _i32(t.amap[1]), _i32(t.amap[2]), _f64(t.amap[3])
            vp_ = lambda a: a.ctypes.data_as(C.c_void_p)
            rc = self.lib.dsp_lp_template_set_matrix_params(h, len(ar), vp_(ar), vp_(ac), vp_(ak), vp_(av))
            if rc != 0:
                raise RuntimeError(f"dsp_lp_template_set_matrix_params failed ({rc}): {self.lib.dsp_lp_last_error().decode()}")
        self.opts = _Opts()
        self.lib.dsp_lp_default_opts(C.byref(self.opts))
        self.opts.tol, self.opts.feas_tol, self.opts.max_iter, self.opts.step_frac = tol, feas_tol, max_iter, step_frac
        self.opts.kernel = kernel
        # proximal term: the library default (1e-8) unless the caller or the template asks otherwise (a template whose feasible set has
        # no strict interior, e.g. templates.solar_battery_hydrogen, records the value its LPs converge with)
        self.opts.reg_primal = float(template.meta.get("reg_primal", 1e-8) if reg_primal is None else reg_primal)
        st = t.meta.get("stage_wb")
        self.has_stage = False
        if st is not None and kernel not in (KERNEL_BAND, KERNEL_DENSE):
            ci, ri = _i32(st["col_idx"]), _i32(st["row_idx"])
            sd = _StageWB(T=st["T"], a=st["a"], binv=st["binv"], half=st["half"], delta=st["delta"], dur=st["dur"],
                          k_rev=st["k_rev"], wcf_off=st["wcf_off"], p_off=st["p_off"],
                          col_idx=ci.ctypes.data_as(C.c_void_p), row_idx=ri.ctypes.data_as(C.c_void_p))
            self._check(self.lib.dsp_lp_template_set_stage_wb(self.handle, C.byref(sd)), "dsp_lp_template_set_stage_wb")
            self.has_stage = True
        # descriptor-driven stage kernel for templates of the single-storage-chain family (structure found on the template itself)
        self.has_chain1 = False
        if st is None and kernel not in (KERNEL_BAND, KERNEL_DENSE) and t.m <= 96:
            from .lp_template import detect_chain1
            d1 = detect_chain1(t)
            if d1 is not None:
                ci, ri, cf, cn = _i32(d1["col_idx"]), _i32(d1["row_idx"]), _f64(d1["coef"]), _f64(d1["coef_next"])
                sd = _StageChain1(T=d1["T"], NF=d1["NF"], col_idx=ci.ctypes.data_as(C.c_void_p), row_idx=ri.ctypes.data_as(C.c_void_p),
                                  coef=cf.ctypes.data_as(C.c_void_p), coef_next=cn.ctypes.data_as(C.c_void_p))
                self._check(self.lib.dsp_lp_template_set_stage_chain1(self.handle, C.byref(sd)), "dsp_lp_template_set_stage_chain1")
                self.has_chain1 = True

    def close(self):
        if getattr(self, "handle", None):
            self.lib.dsp_lp_template_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.dsp_lp_last_error().decode()}")

    # ------------------------------------------------------------------ device tensors
    def solve(self, cparams, rparams=None, want_x=False, want_y=False, out=None):
        """cparams: cuda float64 [N,Pc]; rparams: cuda float64 [N,Pr] or [Pr] (shared by the batch).
        Stream-ordered on torch's current stream, no synchronisation."""
        import torch
        t = self.t
        if not torch.is_tensor(cparams) or not cparams.is_cuda or cparams.dtype != torch.float64:
            raise ValueError("cparams must be a CUDA float64 tensor (no CPU path)")
        if cparams.dim() != 2 or cparams.shape[1] != t.Pc:
            raise ValueError(f"cparams must have shape [N, {t.Pc}], got {tuple(cparams.shape)}")
        cparams = cparams.contiguous()
        N = cparams.shape[0]
        dev = cparams.device
        rstride = 0
        rptr = None
        if t.Pr:
            if rparams is None or not torch.is_tensor(rparams) or not rparams.is_cuda or rparams.dtype != torch.float64 \
                    or rparams.device != dev:
                raise ValueError(f"rparams must be a CUDA float64 tensor on {dev} (template has Pr = {t.Pr})")
            if tuple(rparams.shape) not in ((t.Pr,), (N, t.Pr)):
                raise ValueError(f"rparams must have shape [{t.Pr}] or [{N}, {t.Pr}], got {tuple(rparams.shape)}")
            rparams = rparams.contiguous()
            rstride = 0 if rparams.dim() == 1 else t.Pr
            rptr = rparams.data_ptr()
        if out is not None:
            self._check_out(out, N, want_x, want_y, lambda a, shape, dt: torch.is_tensor(a) and a.is_cuda and a.device == dev
                            and a.is_contiguous() and tuple(a.shape) == shape and a.dtype == {"f8": torch.float64, "i4": torch.int32}[dt])
        if out is None:
            out = LPResult(torch.empty(N, dtype=torch.float64, device=dev),
                           torch.empty(N, dtype=torch.int32, device=dev),
                           torch.empty(N, dtype=torch.int32, device=dev),
                           torch.empty((N, t.n), dtype=torch.float64, device=dev) if want_x else None,
                           torch.empty((N, t.m), dtype=torch.float64, device=dev) if want_y else None)
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.dsp_lp_solve_batch(self.handle, N, cparams.data_ptr(), rptr, rstride, C.byref(self.opts),
                                         out.obj.data_ptr(), out.status.data_ptr(), out.iters.data_ptr(),
                                         out.x.data_ptr() if out.x is not None else None,
                                         out.y.data_ptr() if out.y is not None else None, C.c_void_p(stream))
        self._check(rc, "dsp_lp_solve_batch")
        return out

    # ------------------------------------------------------------------ host arrays (copies included)
    def solve_host(self, cparams, rparams=None, want_x=False, want_y=False, out=None):
        """numpy in / numpy out through dsp_lp_solve_batch_host.  Page-locked arrays (see ``pinned_empty``) skip the
        library's staging copy; ``out`` = a previous LPResult of the same shape is reused (no allocation)."""
        t = self.t
        cparams = _f64(np.atleast_2d(cparams))
        if cparams.ndim != 2 or cparams.shape[1] != t.Pc:
            raise ValueError(f"cparams must have shape [N, {t.Pc}], got {cparams.shape}")
        N = cparams.shape[0]
        rstride, rptr = 0, None
        if t.Pr:
            if rparams is None:
                raise ValueError(f"rparams is required (template has Pr = {t.Pr})")
            rparams = _f64(rparams)
            if rparams.shape not in ((t.Pr,), (N, t.Pr)):
                raise ValueError(f"rparams must have shape [{t.Pr}] or [{N}, {t.Pr}], got {rparams.shape}")
            rstride = 0 if rparams.ndim == 1 else t.Pr
            rptr = rparams.ctypes.data_as(C.c_void_p)
        if out is not None:
            self._check_out(out, N, want_x, want_y, lambda a, shape, dt: isinstance(a, np.ndarray) and a.flags.c_contiguous
                            and a.shape == shape and a.dtype == np.dtype(dt))
            obj, status, iters, x, y = out.obj, out.status, out.iters, out.x, out.y
        else:
            obj = np.empty(N); status = np.empty(N, np.int32); iters = np.empty(N, np.int32)
            x = np.empty((N, t.n)) if want_x else None
            y = np.empty((N, t.m)) if want_y else None
        vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
        rc = self.lib.dsp_lp_solve_batch_host(self.handle, N, vp(cparams), rptr, rstride, C.byref(self.opts),
                                              vp(obj), vp(status), vp(iters), vp(x), vp(y))
        self._check(rc, "dsp_lp_solve_batch_host")
        return LPResult(obj, status, iters, x, y)

    def _check_out(self, out, N, want_x, want_y, ok):
        """a reused LPResult must match the batch: a wrong shape / dtype would be an out-of-bounds device write"""
        t = self.t
        if not (ok(out.obj, (N,), "f8") and ok(out.status, (N,), "i4") and ok(out.iters, (N,), "i4")):
            raise ValueError(f"out.obj / out.status / out.iters must be contiguous [{N}] float64 / int32 / int32 buffers")
        if (out.x is not None and not ok(out.x, (N, t.n), "f8")) or (out.y is not None and not ok(out.y, (N, t.m), "f8")):
            raise ValueError(f"out.x / out.y must be contiguous float64 [{N}, {t.n}] / [{N}, {t.m}]")
        if (want_x and out.x is None) or (want_y and out.y is None):
            raise ValueError("want_x / want_y set but the reused LPResult has no x / y buffer")

    @staticmethod
    def pinned_empty(shape, dtype=np.float64):
        """page-locked numpy array (backed by a pinned torch tensor): host buffers the C ABI can DMA from/to directly"""
        import torch
        tt = torch.empty(shape, dtype={np.float64: torch.float64, np.int32: torch.int32}[np.dtype(dtype).type]).pin_memory()
        return tt.numpy()          # the array keeps the pinned tensor alive (ndarray.base)

    # ------------------------------------------------------------------
    def to_model_space(self, x):
        """template-space primal -> the reference model's Var values (lower-bound shift, column scaling)."""
        return x * self.t.col_scale + self.t.col_shift
