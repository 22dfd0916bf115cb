"""per-phase cycle split of a round of the generation-2 stage kernel on C2 (10 000 LPs, T = 24), at 8 and at 4 warps per SM

needs a -DDSP_PHASES build of the library, named by DSP_LP_LIB:
    nvcc <NVCC_FLAGS of dispatches_b200/csrc/build.py> -DDSP_PHASES dispatches_b200/csrc/dsp_lp.cu -o build/phases/libdsp_lp.so
    DSP_LP_LIB=$PWD/build/phases/libdsp_lp.so python tools/gpu_stage2_phases.py [--pass2-twice] [--compare DIR] [warps ...]
The counters (dsp_stage2.cuh) sum over warp 0 of every CTA; 8 warps per SM are two per scheduler, 4 are one.  Only this
instrumentation build reads DSP_STAGE2_WARPS (the product library reads no environment), so the 8- vs 4-warp comparison runs
with the counters compiled in.

--pass2-twice runs pass 2 twice back to back in every round (DSP_STAGE2_PASS2_TWICE, instrumentation build only) and reports
the two copies apart: the second runs instructions the first has just fetched, so the difference is the first copy's fetch
cost.  Results must not change: --compare DIR checks obj / status / iters of every run against `bench.py --dump-outputs DIR`
of the product build (the same C2 batch).
"""
import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, ".")
import numpy as np

from dispatches_b200 import scenarios as SC, solver as S, templates as TP

NAMES = ["convergence check", "refill", "pass 1", "factor + predictor solve", "pass 2", "pass 3 + corrector solve",
         "pass 4", "pass 5", "exit vote"]
ap = argparse.ArgumentParser()
ap.add_argument("warps", nargs="*", default=["8", "4"])
ap.add_argument("--pass2-twice", action="store_true")
ap.add_argument("--compare", metavar="DIR")
args = ap.parse_args()
lib = S.load_library()
if not hasattr(lib, "dsp_lp_phases"):
    raise SystemExit(f"{S._LIB_PATH} is not a -DDSP_PHASES build")
if args.pass2_twice:
    os.environ["DSP_STAGE2_PASS2_TWICE"] = "1"


def phases(reset=True):
    buf = (C.c_ulonglong * 16)()
    lib.dsp_lp_phases(buf, 1 if reset else 0)
    return np.array(list(buf), float)


lmp, cf, W, P = SC.c2(10000)
rp = TP.wind_battery_rparams(24, cf, W, P)[0]
sol = S.BatchLPSolver(TP.wind_battery(24), kernel=S.KERNEL_STAGE)
ref = {k: np.load(os.path.join(args.compare, k + ".npy")) for k in ("obj", "status", "iters")} if args.compare else None
reps = 5
for w in args.warps:
    os.environ["DSP_STAGE2_WARPS"] = w
    sol.solve_host(lmp, rp)                       # warm-up
    phases()
    for _ in range(reps):
        r = sol.solve_host(lmp, rp)
    ph = phases()
    launch = S.last_launch()
    rounds, idle, late = ph[9], ph[12], ph[13]
    body = ph[:9].sum() + ph[14]
    print(f"== {w} warps per SM  launch {launch}  iters mean {r.iters.mean():.2f}  non-optimal {int((r.status != 0).sum())}")
    print(f"   warp 0 of each CTA, per launch: rounds run {rounds / reps:.0f}, after the counter ran dry {late / reps:.0f},"
          f" rounds waited out of work {idle / reps:.0f}")
    print(f"   cycles per round run (all phases) {body / rounds:.0f}")
    for k, nm in enumerate(NAMES):
        print(f"   {nm:26s} {ph[k] / rounds:8.0f} cycles/round  {100 * ph[k] / body:5.1f} %")
        if k == 4 and args.pass2_twice:
            print(f"   {'pass 2, second copy':26s} {ph[14] / rounds:8.0f} cycles/round  {100 * ph[14] / body:5.1f} %"
                  f"  (first copy - second: {(ph[4] - ph[14]) / rounds:.0f})")
    print(f"   share of warp 0's time after the ticket counter ran dry: {100 * ph[10] / ph[11]:.1f} %"
          f"  (per CTA {ph[11] / reps:.3g} cycles summed over CTAs)")
    if ref is not None:
        same = {k: bool(np.array_equal(np.asarray(getattr(r, k), np.float64), ref[k])) for k in ref}
        print(f"   obj / status / iters bitwise equal to {args.compare}: {same}")
    sys.stdout.flush()
