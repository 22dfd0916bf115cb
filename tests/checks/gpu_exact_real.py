"""All 10 000 C2 LPs and the strided C5 sample (tests/real_lps.py) on the GPU through check_exact's measures, on their usual kernel
(stage 2) and on the dense kernel (DSP_KERNEL_DENSE), the PV + battery + hydrogen design LPs (baked and with a PV series per LP)
at T = 24 and 48 on the dense kernel and the dense cluster kernel, and at T = 72, 96 and 168 on the dense cluster kernel: prints, per
run, how many LPs ended OPTIMAL and the largest error of every measure, and exits non-zero if any LP is not OPTIMAL or over a bar.

    python tests/checks/gpu_exact_real.py [--procs P]

Exact certification (about 7 ms per 24-hour dispatch LP, and on one core 0.2 to 2 s per design LP at T = 24 and 48, 2 to 6 s at
T = 72, about 30 s at T = 96 and 40 to 80 s at T = 168) and the per-LP KKT residuals run in P worker processes."""
import argparse
import multiprocessing as mp
import sys
import time
from pathlib import Path

import numpy as np

sys.path[:0] = [str(Path(__file__).resolve().parents[1]), str(Path(__file__).resolve().parents[2])]
import real_lps as R                                      # noqa: E402
from dispatches_b200 import scenarios as SC               # noqa: E402
from dispatches_b200 import solver as S                   # noqa: E402
from dispatches_b200 import templates as TP               # noqa: E402
from oracle.highs import host_cores                       # noqa: E402

_JOB = {}


def _errors(k):
    s, r = _JOB["s"], _JOB["r"]
    return R.errors(s.take(k), r.obj[k], r.x[k], r.y[k])


def _sets(procs):
    """(name, a function that certifies the set, kernels to run it on)"""
    def c2():
        lmp, cf, W, P = SC.c2()
        return R.certify(TP.wind_battery(24), lmp, TP.wind_battery_rparams(24, cf, W, P), procs=procs)

    def c5():
        lmp, cf, W, P = SC.c5()
        k = np.arange(0, len(lmp), R.C5_STRIDE)
        return R.certify(TP.wind_battery(24), lmp[k], TP.wind_battery_rparams(24, cf[k], W[k], P[k]), procs=procs)

    yield "C2", c2, (S.KERNEL_AUTO, S.KERNEL_DENSE)
    yield "C5", c5, (S.KERNEL_AUTO,)
    for T, N in ((24, 256), (48, 64), (72, 64), (96, 32), (168, 12)):
        kernels = (S.KERNEL_DENSE, S.KERNEL_DENSE_CLUSTER) if 15 * T + 3 <= 1024 else (S.KERNEL_DENSE_CLUSTER,)
        yield f"solar_design{T}", lambda T=T, N=N: R.solar_design(T, N, procs=procs), kernels
        yield f"solar_design_pv{T}", lambda T=T, N=N: R.solar_design_pv(T, N, procs=procs), kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=host_cores())
    a = ap.parse_args()
    bad = 0
    for set_name, make, kernels in _sets(a.procs):
        t0 = time.perf_counter()
        s = make()
        t1 = time.perf_counter()
        for kernel in kernels:
            name = set_name + {S.KERNEL_DENSE: " on the dense kernel",
                               S.KERNEL_DENSE_CLUSTER: " on the dense cluster kernel"}.get(kernel, "")
            bad += _check(name, s, S.BatchLPSolver(s.t, kernel=kernel), a.procs, t1 - t0)
    return 1 if bad else 0


def _check(name, s, sol, procs, cert_s):
    r = sol.solve_host(s.cparams, s.rparams, want_x=True, want_y=True)
    _JOB.update(s=s, r=r)
    chunks = np.array_split(np.arange(len(s)), 4 * procs)
    with mp.get_context("fork").Pool(procs) as pool:
        es = pool.map(_errors, chunks)
    worst = {key: max((e[key] for e in es if e[key] is not None), default=None) for key in es[0]}
    opt = int((r.status == S.OPTIMAL).sum())
    print(f"{name}: {opt} / {len(s)} OPTIMAL, {int(s.unique_x.sum())} unique in x, {int(s.unique_y.sum())} in y, "
          f"{int((s.lp_mag == 0).sum())} with a zero LP part, {int((s.pivots > 0).sum())} repaired (at most {int(s.pivots.max())} "
          f"pivots), certified in {cert_s:.0f} s; largest errors {R.fmt(worst)}", flush=True)
    z = lambda v: 0.0 if v is None else v
    ok = (opt == len(s) and worst["obj"] <= R.OBJ_REL and z(worst["lp"]) <= R.OBJ_REL
          and max(z(worst[k]) for k in ("x", "y", "fixed", "inside")) <= R.XY_REL
          and max(worst["primal"], worst["bound"]) <= R.KKT_PRIMAL and z(worst["dual_inf"]) <= R.KKT_DUAL
          and z(worst["gap"]) <= R.KKT_GAP)
    if not ok:
        print(f"{name}: over a bar", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
