"""Throughput of the dense cluster kernel on the PV + battery + hydrogen design LP, next to the single-CTA dense kernel at T = 48 and to
HiGHS at T = 168: kernel time from CUDA events after a warm-up launch (best of three), LPs/s, iterations, non-optimal count, the FP64
rate from the algorithmic count of gpu_dense_check.py, the workspace bytes the factorisation moves by the kernel's schedule, the
cluster size and clusters in flight, and the card's name, power limit and max SM clock, all in one run.

    python tests/checks/gpu_dense_cluster_check.py [--out DIR]

Workspace bytes of one factorisation (nt tile rows of 64, C ranks, kGroup = 2 target tiles per group, 32 KB per tile): every target tile
(I, J) is read and written once; per group of target tiles, W(J, K) and the group's W(I, K) are read for every K < J; the panel sweep
reads L_JJ once per rank with panel tiles and reads / writes each panel tile once.
"""
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

sys.path.insert(0, ".")
sys.path.insert(0, "tests/checks")
import numpy as np
import torch

from dispatches_b200 import scenarios as SC, solver as S, templates as TP
from oracle import highs as H, lp_models as L

TILE_BYTES = 64 * 64 * 8
GROUP = 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def factor_bytes(nt, C):
    tiles = 0
    for J in range(nt):
        for r in range(C):
            own = list(range(J + ((r - J % C) % C + C) % C, nt, C))
            for g0 in range(0, len(own), GROUP):
                ng = min(GROUP, len(own) - g0)
                tiles += 2 * ng + J * (1 + ng)
            below = [I for I in own if I > J]
            if below:
                tiles += 1 + 2 * len(below)
    return tiles * TILE_BYTES


def batch(T, N, seed):
    """T = 168: the year's 52 weeks of day-ahead prices, repeated with seeded lognormal perturbations beyond 52 LPs; else N random
    windows of the year"""
    year = SC.pool()["pq1000_da_lmp"][:8736]
    rng = np.random.default_rng(seed)
    if T == 168:
        lmp = np.vstack([year.reshape(52, 168)] * -(-N // 52))[:N]
        lmp[52:] *= rng.lognormal(0, 0.2, lmp[52:].shape)
    else:
        lmp = np.stack([year[s:s + T] for s in rng.integers(0, 8736 - T, N)])
    return lmp, np.tile(L.solar_default_series()["pv_cfs"], T // 24)


def run(T, N, kernel, seed=0):
    lmp, cfs = batch(T, N, seed)
    t = TP.solar_battery_hydrogen_design(T, cfs, reserve_mw=np.full(T, 100.0))
    sol = S.BatchLPSolver(t, kernel=kernel)
    cp = torch.tensor(lmp, device="cuda"); rp = torch.tensor(np.full((N, T), 100e3), device="cuda")
    out = sol.solve(cp, rp)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(3):
        e0.record(); sol.solve(cp, rp, out=out); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    ll = S.last_launch()
    ms = min(ms)
    iters = out.iters.cpu().numpy(); status = out.status.cpu().numpy()
    nt = -(-t.m // 64); mp = 64 * nt
    Ad = abs(t.A).tocsc()
    nterms = int(sum(c * (c + 1) // 2 for c in np.diff(Ad.indptr)))
    flops = float(iters.sum()) * (mp ** 3 / 3 + 2 * nterms + 4 * mp ** 2)
    res = dict(T=T, N=N, m=t.m, kernel="dense_cluster" if kernel == S.KERNEL_DENSE_CLUSTER else "dense", kernel_ms=round(ms, 2),
               lps_per_s=round(N / ms * 1e3, 2), iters_mean=round(float(iters.mean()), 2), iters_max=int(iters.max()),
               non_optimal=int((status != S.OPTIMAL).sum()), fp64_tflops=round(flops / (ms * 1e-3) / 1e12, 3), launch=ll)
    if kernel == S.KERNEL_DENSE_CLUSTER:
        C = ll["problems_per_cta"]
        fb = factor_bytes(nt, C) * float(iters.sum())
        res.update(cluster_size=C, clusters_in_flight=ll["grid"] // C, factor_ws_gb_per_lp=round(fb / N / 1e9, 2),
                   factor_ws_tb_per_s=round(fb / (ms * 1e-3) / 1e12, 3))
    return res, lmp, cfs


def _highs_one(args):
    lmp, cfs, T = args
    return H.solve(L.solar_battery_hydrogen_raw(lmp, True, dict(pv_mw=0.0, turb_mw=0.0), pv_cfs=cfs, load_mw=np.full(T, 100.0),
                                                reserve_mw=np.full(T, 100.0)))[0]


def main():
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    lines = [dict(card=card(), fp64_fma_peak_tflops=round(S.fp64_peak_tflops(), 2))]
    print(json.dumps(lines[0]), flush=True)
    for T, N, k in [(48, 416, S.KERNEL_DENSE), (48, 416, S.KERNEL_DENSE_CLUSTER), (96, 416, S.KERNEL_DENSE_CLUSTER),
                    (168, 52, S.KERNEL_DENSE_CLUSTER), (168, 416, S.KERNEL_DENSE_CLUSTER)]:
        res, lmp, cfs = run(T, N, k)
        lines.append(res)
        print(json.dumps(res), flush=True)
    # HiGHS on the 52 week-long LPs, one per process over every host core
    lmp, cfs = batch(168, 52, 0)
    ncpu = os.cpu_count()
    t0 = time.perf_counter()
    with ProcessPoolExecutor(ncpu) as ex:
        list(ex.map(_highs_one, [(lmp[k], cfs, 168) for k in range(52)]))
    dt = time.perf_counter() - t0
    h = dict(highs_T=168, N=52, host_cores=ncpu, highs_lps_per_s=round(52 / dt, 2))
    lines.append(h)
    print(json.dumps(h), flush=True)
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "dense_cluster_check.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
