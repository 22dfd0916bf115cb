"""Time the crossover (dsp_lp_crossover) against the solve that produced its input, with CUDA events, on one GPU:
C2 (10 000 LPs), C3 (5 000), the 48-hour day-ahead bidder (1 000), the PV + battery + hydrogen design at T = 24 (512) and C4 (2 000).
Prints one JSON line per workload (times, pivots per LP, statuses, placement) and the card and its power limit read in the same run.

    python tests/checks/gpu_crossover_bench.py
"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from dispatches_b200 import scenarios as SC, solver as S, templates as TP  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0) + ", power limit not read"


def workloads():
    rng = np.random.default_rng(5)
    lmp, cf, W, P = SC.c2()
    yield "C2", TP.wind_battery(24), lmp, TP.wind_battery_rparams(24, cf, W, P), {}
    yield "C3", TP.nuclear(48), SC.c3(5000), None, {}
    T, N = 48, 1000
    p = SC.pool()
    idx = rng.integers(0, len(p["dalmp_303"]) - T, N)[:, None] + np.arange(T)[None, :]
    da = p["dalmp_303"][idx]; rt = da * rng.lognormal(0.0, 0.2, (N, T))
    rp = TP.wind_battery_operation_rparams(T, p["dacf_303"][idx], 200.0, 25.0, 100.0, rng.uniform(0, 90000, N), rng.uniform(0, 5000, N), None)
    yield "bidder_48h", TP.wind_battery_operation(T, "bidder_da"), np.concatenate([da, rt, np.full((N, 1), 1e3)], 1), rp, dict(kernel=S.KERNEL_BAND)
    import real_lps as R
    lmp0, d = R._solar_reference()
    N = 512
    lmp = lmp0[None] * rng.lognormal(0.0, 0.3, (N, 24)); load = 1e3 * d["load_mw"][None] * rng.uniform(0.7, 1.2, (N, 24))
    yield "pv_design_24", TP.solar_battery_hydrogen_design(24, d["pv_cfs"]), lmp, load, dict(kernel=S.KERNEL_DENSE)
    yield "C4", TP.fossil_surrogate(168), SC.c4(2000), None, {}


def timed(fn, reps=3):
    ts = []
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); out = fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return out, float(np.median(ts))


def main():
    S.load_library()
    print(json.dumps(dict(card=card())), flush=True)
    for name, t, cp, rp, kw in workloads():
        sol = S.BatchLPSolver(t, **kw)
        cpd = torch.as_tensor(np.ascontiguousarray(cp), device="cuda")
        if t.Pr and np.ndim(rp) == 2 and len(rp) == 1:
            rp = rp[0]                           # one rparams row shared by the batch
        rpd = torch.as_tensor(np.ascontiguousarray(rp), device="cuda") if t.Pr else None
        r, t_solve = timed(lambda: sol.solve(cpd, rpd, want_x=True, want_y=True))
        v, t_x = timed(lambda: sol.crossover(cpd, rpd, r), reps=1 if name == "C4" else 3)
        launch = S.last_launch()
        st, xs, pv = r.status.cpu().numpy(), v.status.cpu().numpy(), v.pivots.cpu().numpy()
        ok = xs == 0
        print(json.dumps(dict(workload=name, N=len(st), m=t.m, n=t.n, solve_ms=round(t_solve, 2), crossover_ms=round(t_x, 2),
                              ratio=round(t_x / t_solve, 2), solve_optimal=int((st == 0).sum()), crossover_optimal=int(ok.sum()),
                              crossover_status=dict(zip(*[a.tolist() for a in np.unique(xs, return_counts=True)])),
                              pivots_mean=round(float(pv[ok].mean()), 2) if ok.any() else None, pivots_max=int(pv[ok].max()) if ok.any() else None,
                              placement="shared memory" if launch["smem_bytes"] > 0 else "workspace", launch=launch)), flush=True)


if __name__ == "__main__":
    main()
