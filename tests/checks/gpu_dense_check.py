"""Throughput of the dense kernel on the PV + battery + hydrogen design LP (pv_battery_hydrogen_design_optimize's template): kernel time
from CUDA events after a warm-up launch, LPs/s, iterations, non-optimal count, the achieved FP64 rate from the algorithmic count
below, the card's name and power limit, and HiGHS on one CPU core for a sample of the same LPs.

    python tests/checks/gpu_dense_check.py [T=24:4096,48:1024]

FP64 count per IPM iteration of an LP (padded size mp = 64 * ceil(m / 64)): mp^3 / 3 for the factorisation, 2 per product of the
assembly list, 2 * 2 mp^2 for the two substitutions (predictor, corrector); the element-wise and CSR passes are left out.
"""
import json
import subprocess
import sys
import time

sys.path.insert(0, ".")
import numpy as np
import torch

from dispatches_b200 import solver as S, templates as TP
from oracle import highs as H, lp_models as L


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def batch(T, N, seed=0):
    d = L.solar_default_series()
    rng = np.random.default_rng(seed)
    lmp0 = np.tile(json.load(open("tests/golden/solar_golden.json"))["lmp_24"], T // 24)
    lmp = lmp0[None] * rng.lognormal(0, 0.3, (N, T))
    load = 100.0 * rng.uniform(0.7, 1.2, (N, T))
    return lmp, load, np.tile(d["pv_cfs"], T // 24)


def run(T, N, reps=3):
    lmp, load, cfs = batch(T, N)
    t = TP.solar_battery_hydrogen_design(T, cfs)
    sol = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE)
    cp = torch.tensor(lmp, device="cuda"); rp = torch.tensor(load * 1e3, device="cuda")
    out = sol.solve(cp, rp)                                      # warm-up (workspace allocation)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        e0.record(); sol.solve(cp, rp, out=out); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    launch = S.last_launch()
    ms = min(ms)
    iters = out.iters.cpu().numpy(); status = out.status.cpu().numpy()
    mp = 64 * -(-t.m // 64)
    Ad = abs(t.A).tocsc()
    nterms = int(sum(c * (c + 1) // 2 for c in np.diff(Ad.indptr)))
    flop_iter = mp ** 3 / 3 + 2 * nterms + 4 * mp ** 2
    flops = float(iters.sum()) * flop_iter
    # HiGHS (one core) on a sample of the same LPs, raw oracle LP
    k = 16
    t0 = time.perf_counter()
    for i in range(k):
        H.solve(L.solar_battery_hydrogen_raw(lmp[i], True, dict(pv_mw=0.0, turb_mw=0.0), pv_cfs=cfs, load_mw=load[i], reserve_mw=np.full(T, 100.0)))
    highs_ms = (time.perf_counter() - t0) / k * 1e3
    return dict(T=T, N=N, m=t.m, n=t.n, w=t.w, kernel_ms=round(ms, 3), lps_per_s=round(N / ms * 1e3, 1), iters_mean=round(float(iters.mean()), 2),
                iters_max=int(iters.max()), non_optimal=int((status != S.OPTIMAL).sum()), fp64_tflops=round(flops / (ms * 1e-3) / 1e12, 3),
                gflop_per_lp=round(flops / N / 1e9, 3), launch=launch, highs_ms_per_lp=round(highs_ms, 2))


if __name__ == "__main__":
    spec = sys.argv[1] if len(sys.argv) > 1 else "24:4096,48:1024"
    print(json.dumps(dict(card=card(), fp64_fma_peak_tflops=round(S.fp64_peak_tflops(), 2))))
    for item in spec.split(","):
        T, N = map(int, item.split(":"))
        print(json.dumps(run(T, N)))
