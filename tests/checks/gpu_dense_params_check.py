"""Cost of per-problem matrix coefficients on the dense kernel: the PV + battery + hydrogen design LP with a PV series per scenario
(templates.solar_battery_hydrogen_design(T, None): each CTA derives its LP's A, A' and assembly products at LP load) against the same
LPs through per-series baked templates.  Kernel time from CUDA events after a warm-up launch, LPs/s, iterations, non-optimal count,
the extra workspace per CTA, the card's name and power limit.

    python tests/checks/gpu_dense_params_check.py [T=24:4096,48:1024] [--series K]

The batch draws K PV series (default 8; PV on a 1/1024 grid, so both paths solve the same LPs bit for bit) and assigns them to the
scenarios round robin; the baked path solves each series' scenarios in one launch of that series' template, and its time is the sum.
"""
import argparse
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np
import torch

from dispatches_b200 import solver as S, templates as TP
from oracle import lp_models as L


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def batch(T, N, K, seed=0):
    d = L.solar_default_series()
    rng = np.random.default_rng(seed)
    lmp = np.tile(json.load(open("tests/golden/solar_golden.json"))["lmp_24"], T // 24)[None] * rng.lognormal(0, 0.3, (N, T))
    load = 100.0 * rng.uniform(0.7, 1.2, (N, T))
    series = np.maximum(np.round(np.tile(d["pv_cfs"], T // 24)[None] * rng.uniform(0.5, 1.0, (K, T)) * 1024) / 1024, 1.0 / 1024)
    return lmp, load, series, np.arange(N) % K


def timed(fn, reps=3):
    fn()                                                          # warm-up (workspace allocation)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return min(ms)


def run(T, N, K):
    lmp, load, series, which = batch(T, N, K)
    reserve = np.full(T, 100.0)
    tp = TP.solar_battery_hydrogen_design(T, None)
    per = S.BatchLPSolver(tp, kernel=S.KERNEL_DENSE)
    cp = torch.tensor(lmp, device="cuda")
    rp = torch.tensor(TP.solar_design_rparams(T, load, series[which], reserve), device="cuda")
    out = per.solve(cp, rp)
    ms_per = timed(lambda: per.solve(cp, rp, out=out))
    launch = S.last_launch()
    parts = []
    for k in range(K):
        sel = np.flatnonzero(which == k)
        sol = S.BatchLPSolver(TP.solar_battery_hydrogen_design(T, series[k], reserve_mw=reserve), kernel=S.KERNEL_DENSE)
        c = torch.tensor(lmp[sel], device="cuda"); r = torch.tensor(load[sel] * 1e3, device="cuda")
        o = sol.solve(c, r)
        parts.append((sol, c, r, o, sel))
    ms_baked = timed(lambda: [p[0].solve(p[1], p[2], out=p[3]) for p in parts])
    it_b = np.empty(N, np.int32); st_b = np.empty(N, np.int32); obj_b = np.empty(N)
    for sol, c, r, o, sel in parts:
        it_b[sel] = o.iters.cpu().numpy(); st_b[sel] = o.status.cpu().numpy(); obj_b[sel] = o.obj.cpu().numpy()
    it = out.iters.cpu().numpy(); st = out.status.cpu().numpy(); obj = out.obj.cpu().numpy()
    Ad = abs(tp.A).tocsc()
    nterms = int(sum(c * (c + 1) // 2 for c in np.diff(Ad.indptr)))
    extra = 2 * tp.A.nnz + nterms
    return dict(T=T, N=N, series=K, m=tp.m, n=tp.n, nnz=int(tp.A.nnz), assembly_products=nterms,
                extra_workspace_per_cta_kb=round(extra * 8 / 1024, 1), tiles_per_cta_kb=round((-(-tp.m // 64)) * (-(-tp.m // 64) + 1) / 2 * 64 * 64 * 8 / 1024, 1),
                per_problem=dict(kernel_ms=round(ms_per, 3), lps_per_s=round(N / ms_per * 1e3, 1), iters_mean=round(float(it.mean()), 2),
                                 iters_max=int(it.max()), non_optimal=int((st != S.OPTIMAL).sum()), launch=launch),
                baked=dict(launches=K, ms=round(ms_baked, 3), lps_per_s=round(N / ms_baked * 1e3, 1), iters_mean=round(float(it_b.mean()), 2),
                           iters_max=int(it_b.max()), non_optimal=int((st_b != S.OPTIMAL).sum())),
                slowdown=round(ms_per / ms_baked, 4), bitwise_equal_obj=bool(np.array_equal(obj, obj_b)),
                bitwise_equal_iters=bool(np.array_equal(it, it_b)))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("spec", nargs="?", default="24:4096,48:1024")
    ap.add_argument("--series", type=int, default=8)
    a = ap.parse_args()
    print(json.dumps(dict(card=card())))
    for item in a.spec.split(","):
        T, N = map(int, item.split(":"))
        print(json.dumps(run(T, N, a.series)))
