"""Time the parametric walk (dsp_lp_parametric) against the solve and the crossover that produce its input, with CUDA events, on one
GPU: C2 (10 000 LPs) along the battery size from 0 MW to +inf and along its 24 LMP axes, C3 (5 000) along its 48 LMP axes, the 48-hour
day-ahead bidder (1 000) along its 48 day-ahead LMP axes, and the PV + battery + hydrogen design at T = 24 (512) along the load of
every hour scaled together; and, for comparison, the interior-point solves of the same C2 batch at C5's 8 battery ratios.  Prints one
JSON line per workload (times, walks, events per walk, statuses, placement) and the card, its power limit and SM clock read in the
same run.

    python tests/checks/gpu_parametric_bench.py
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "checks"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from dispatches_b200 import scenarios as SC, solver as S, templates as TP  # noqa: E402
from gpu_crossover_bench import timed, workloads  # noqa: E402
from gpu_ranging_bench import card  # noqa: E402


def _axes(P, q):
    d = np.zeros((len(q), P))
    d[np.arange(len(q)), q] = 1.0
    return d


def cases():
    w = {name: (t, cp, rp, kw) for name, t, cp, rp, kw in workloads() if name != "C4"}
    lmp, cf, W, _ = SC.c2()
    t = TP.wind_battery(24)
    dr = np.zeros((1, t.Pr)); dr[0, 24] = 1e3
    yield "C2_battery_from_0", t, lmp, TP.wind_battery_rparams(24, cf, W, 0.0), {}, None, dr, 512
    t, cp, rp, kw = w["C2"]
    yield "C2_lmp_axes", t, cp, rp, kw, _axes(t.Pc, np.arange(24)), None, 256
    t, cp, rp, kw = w["C3"]
    yield "C3_lmp_axes", t, cp, rp, kw, _axes(t.Pc, np.arange(48)), None, 256
    t, cp, rp, kw = w["bidder_48h"]
    yield "bidder_48h_da_lmp_axes", t, cp, rp, kw, _axes(t.Pc, np.arange(48)), np.zeros((48, t.Pr)), 256
    t, cp, rp, kw = w["pv_design_24"]
    yield "pv_design_24_load", t, cp, rp, kw, np.zeros((1, t.Pc)), None, 256


def main():
    S.load_library()
    print(json.dumps(dict(card=card())), flush=True)
    for name, t, cp, rp, kw, dc, dr, ev in cases():
        sol = S.BatchLPSolver(t, **kw)
        cpd = torch.as_tensor(np.ascontiguousarray(cp), device="cuda")
        if t.Pr and np.ndim(rp) == 2 and len(rp) == 1:
            rp = rp[0]
        rpd = torch.as_tensor(np.ascontiguousarray(rp), device="cuda") if t.Pr else None
        if name == "pv_design_24_load":                        # every hour's load scaled together: d rp = rp of each LP
            dc = torch.zeros((len(cp), 1, t.Pc), dtype=torch.float64, device="cuda")
            dr = rpd[:, None, :].contiguous()
        else:
            dc = torch.as_tensor(dc, device="cuda") if dc is not None else None
            dr = torch.as_tensor(dr, device="cuda") if dr is not None else None
        r, t_solve = timed(lambda: sol.solve(cpd, rpd, want_x=True, want_y=True))
        v, t_x = timed(lambda: sol.crossover(cpd, rpd, r), reps=1)
        g, t_w = timed(lambda: sol.parametric(cpd, rpd, v, dc, dr, max_events=ev), reps=1)
        launch = S.last_launch()
        cnt, st = g.count.cpu().numpy(), g.status.cpu().numpy()
        print(json.dumps(dict(workload=name, N=len(cp), m=t.m, n=t.n, K=int(cnt.shape[1]), walks=int(cnt.size), solve_ms=round(t_solve, 2),
                              crossover_ms=round(t_x, 2), walk_ms=round(t_w, 2), events_mean=round(float(cnt.mean()), 2),
                              events_max=int(cnt.max()), walk_status=dict(zip(*[a.tolist() for a in np.unique(st, return_counts=True)])),
                              placement="shared memory" if launch["smem_bytes"] > 0 else "workspace", launch=launch)), flush=True)
        del g, v, r
        torch.cuda.empty_cache()
    # for comparison: the interior-point solves of the C2 batch at C5's 8 battery ratios
    lmp, cf, W, _ = SC.c2()
    t = TP.wind_battery(24)
    sol = S.BatchLPSolver(t)
    cpd = torch.as_tensor(lmp, device="cuda")
    _, _, W5, P5 = SC.c5()
    ratios = np.unique(np.round(P5 / W5, 9))
    tot = 0.0
    for a in ratios:
        rpd = torch.as_tensor(TP.wind_battery_rparams(24, cf, W, a * W)[0], device="cuda")
        _, ms = timed(lambda: sol.solve(cpd, rpd))
        tot += ms
    print(json.dumps(dict(workload="C2_ipm_at_C5_battery_ratios", N=len(lmp), ratios=len(ratios), solve_ms_total=round(tot, 2))), flush=True)


if __name__ == "__main__":
    main()
