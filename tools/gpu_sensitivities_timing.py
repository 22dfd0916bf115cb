"""Times the sensitivity post-pass (dsp_lp_sensitivities) against the solve that precedes it, with CUDA events, inputs and outputs in
HBM: C2 (10 000 wind + battery LPs, T = 24), C5 (the 560 640-LP design sweep, in chunks) and FY (64 full-year wind + battery LPs,
T = 8736).  Bytes per LP are counted from shapes: status, x, y and the parameter rows read, rc and both gradients written (the
template structure is read once per CTA and not counted).  Prints the card and one table row per workload, and writes the rows as JSON with --out.

    python tools/gpu_sensitivities_timing.py [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from dispatches_b200 import scenarios as SC, solver as S, templates as TP  # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def workload(name, t, cp, rp, chunk, reps_sens=20):
    sol = S.BatchLPSolver(t)
    dev = torch.device("cuda", 0)
    N = cp.shape[0]
    solve_ms = sens_ms = 0.0
    nonopt = 0
    for a in range(0, N, chunk):
        cpt = torch.as_tensor(cp[a:a + chunk], device=dev)
        rpt = torch.as_tensor(rp[a:a + chunk] if rp.ndim == 2 else rp, device=dev)
        out = {}

        def solve():
            out["r"] = sol.solve(cpt, rpt, want_x=True, want_y=True)
        solve_ms += time_ms(solve, 1)
        r = out["r"]
        nonopt += int((r.status != S.OPTIMAL).sum())
        sens_ms += time_ms(lambda: sol.sensitivities(cpt, rpt, r), reps_sens)
        del r, out
    rw = t.Pr if rp.ndim == 2 else 0
    bytes_lp = 4 + 8 * (t.n + t.m + t.Pc + rw) + 8 * (t.n + t.Pc + t.Pr)
    share = bytes_lp * N / (sens_ms * 1e-3) / HBM
    return dict(workload=name, N=N, n=t.n, m=t.m, solve_ms=solve_ms, sens_ms=sens_ms, sens_over_solve=sens_ms / solve_ms,
                bytes_per_lp=bytes_lp, hbm_share=share, non_optimal=nonopt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    rows = []
    lmp, cf, W, P = SC.c2(10000)
    rows.append(workload("C2", TP.wind_battery(24), lmp, TP.wind_battery_rparams(24, cf, W, P)[0], 10000))
    lmp, cf, W, P = SC.c5()
    rows.append(workload("C5", TP.wind_battery(24), lmp, TP.wind_battery_rparams(24, cf, W, P), 140160, reps_sens=5))
    p = SC.pool()
    T = 8736
    lmpf = np.tile(p["dalmp_303"][:T], (64, 1)) * np.random.default_rng(0).lognormal(0, 0.1, (64, 1))
    rows.append(workload("FY", TP.wind_battery(T), lmpf, TP.wind_battery_rparams(T, p["dacf_303"][:T], SC.FIXED_WIND_MW,
                                                                                   0.25 * SC.FIXED_WIND_MW)[0], 64, reps_sens=5))
    c = card()
    print(f"card: {c}")
    print("| workload | LPs | solve (ms) | post-pass (ms) | post-pass / solve | bytes / LP | share of 3.35 TB/s |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['workload']} | {r['N']} | {r['solve_ms']:.2f} | {r['sens_ms']:.3f} | {r['sens_over_solve']:.4f} | {r['bytes_per_lp']} | "
              f"{100 * r['hbm_share']:.1f} % |")
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        json.dump(dict(card=c, rows=rows), open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
