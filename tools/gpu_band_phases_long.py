"""band kernel, workspace placement: per-phase cycles (warp 0 of block 0) on wind_battery_pem(8784) and C4 (fossil_surrogate(168))

needs the -DDSP_PHASES build of the library, named by DSP_LP_LIB (see tools/gpu_stage2_phases.py); the placement is forced with
DSP_BAND_MODE=ws, which only that build reads.

    DSP_LP_LIB=$PWD/build/phases/libdsp_lp.so python tools/gpu_band_phases_long.py
"""
import ctypes as C
import os
import sys

sys.path.insert(0, ".")
import numpy as np
from dispatches_b200 import scenarios as SC, solver as S, templates as TP

lib = S.load_library()
if not hasattr(lib, "dsp_lp_phases"):
    raise SystemExit(f"{S._LIB_PATH} is not a -DDSP_PHASES build")
os.environ["DSP_BAND_MODE"] = "ws"
NAMES = {0: "residuals + scaling d (CSR)", 1: "assembly of M (element-wise)", 2: "factorisation (sweep)",
         3: "Newton predictor (2 CSR + 2 sweeps)", 4: "step lengths + mu_aff", 5: "Newton corrector (2 CSR + 2 sweeps)",
         6: "steps + update", 7: "convergence test / exit"}


def phases():
    buf = (C.c_ulonglong * 16)()
    lib.dsp_lp_phases(buf, 1)
    return np.array(list(buf), float)


p = SC.pool()
T = 8784
lmp, cf = p["pq1000_rt_lmp"][:T], p["pq1000_rt_cf"][:T]
N = 132
cases = {
    "wind_battery_pem(8784)": (TP.wind_battery_pem(T), np.tile(np.concatenate([lmp, [2.5]]), (N, 1)),
                               TP.wind_battery_rparams(T, cf, 847.0, 150.0, pem_mw=200.0)[0]),
    "C4 fossil_surrogate(168)": (TP.fossil_surrogate(168), SC.c4(2000), None),
}
for name, (t, cp, rp) in cases.items():
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
    phases()
    r = sol.solve_host(cp, rp)
    ph = phases()
    tot = ph[:8].sum()
    print(f"{name}: m = {t.m}, w = {t.w}, launch {S.last_launch()}, iterations mean {r.iters.mean():.1f}, "
          f"total {tot:.3e} cycles (warp 0 of block 0)")
    for k, nm in NAMES.items():
        print(f"   {nm:40s} {100 * ph[k] / tot:6.1f} %")
