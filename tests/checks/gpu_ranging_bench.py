"""Time the ranging post-pass (dsp_lp_ranging) against the solve and the crossover that produce its input, with CUDA events, on one
GPU, with the K = Pc + Pr coordinate directions: C2 (10 000 LPs), C3 (5 000), the 48-hour day-ahead bidder (1 000), the PV + battery +
hydrogen design at T = 24 (512) and C4 (2 000).  Prints one JSON line per workload (times, K, statuses, placement) and the card, its
power limit and SM clock read in the same run.

    python tests/checks/gpu_ranging_bench.py
"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "checks"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from dispatches_b200 import solver as S  # noqa: E402
from gpu_crossover_bench import timed, workloads  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0) + ", not read"


def main():
    S.load_library()
    print(json.dumps(dict(card=card())), flush=True)
    for name, t, cp, rp, kw in workloads():
        sol = S.BatchLPSolver(t, **kw)
        cpd = torch.as_tensor(np.ascontiguousarray(cp), device="cuda")
        if t.Pr and np.ndim(rp) == 2 and len(rp) == 1:
            rp = rp[0]
        rpd = torch.as_tensor(np.ascontiguousarray(rp), device="cuda") if t.Pr else None
        r, t_solve = timed(lambda: sol.solve(cpd, rpd, want_x=True, want_y=True))
        v, t_x = timed(lambda: sol.crossover(cpd, rpd, r), reps=1)
        g, t_r = timed(lambda: sol.ranging(cpd, rpd, v), reps=1 if name == "C4" else 3)
        launch = S.last_launch()
        rs = g.status.cpu().numpy()
        print(json.dumps(dict(workload=name, N=len(rs), m=t.m, n=t.n, K=t.Pc + t.Pr, solve_ms=round(t_solve, 2), crossover_ms=round(t_x, 2),
                              ranging_ms=round(t_r, 2), ranging_over_crossover=round(t_r / t_x, 2),
                              ranging_status=dict(zip(*[a.tolist() for a in np.unique(rs, return_counts=True)])),
                              placement="shared memory" if launch["smem_bytes"] > 0 else "workspace", launch=launch)), flush=True)


if __name__ == "__main__":
    main()
