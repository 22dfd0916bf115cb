"""stage kernel generation 2 vs generation 1 vs band kernel: parity + timing on C2 (10 000 LPs) and a C5 slice; other horizons."""
import sys, json
sys.path.insert(0, ".")
import numpy as np, torch
from dispatches_b200 import templates as TP, scenarios as SC, solver as S
dev = torch.device("cuda:0")
out = {}

def timed(sol, cp, rp, reps=9):
    o = sol.solve(cp, rp); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); sol.solve(cp, rp, out=o); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    return o, float(np.median(ts)), float(np.min(ts))

t = TP.wind_battery(24)
v2 = S.BatchLPSolver(t, kernel=S.KERNEL_STAGE); v1 = S.BatchLPSolver(t, kernel=S.KERNEL_STAGE_V1); band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND)
lmp, cf, W, P = SC.c2(10000); rp = TP.wind_battery_rparams(24, cf, W, P)[0]
cp = torch.tensor(lmp, device=dev); rpt = torch.tensor(rp, device=dev)
a, ms2, mn2 = timed(v2, cp, rpt); l2 = S.last_launch()
b, ms1, mn1 = timed(v1, cp, rpt); l1 = S.last_launch()
c = band.solve(cp[:1024], rpt); torch.cuda.synchronize()
ao, bo, co = a.obj.cpu().numpy(), b.obj.cpu().numpy(), c.obj.cpu().numpy()
rel = lambda x, y: float((np.abs(x - y) / np.maximum(1, np.abs(y))).max())
out["C2"] = dict(v2_ms=ms2, v2_min_ms=mn2, v1_ms=ms1, v1_min_ms=mn1, speedup=ms1 / ms2, v2_launch=l2, v1_launch=l1,
                 v2_non_optimal=int((a.status != 0).sum()), iters_v2=float(a.iters.float().mean()), iters_v1=float(b.iters.float().mean()),
                 iters_equal=float((a.iters == b.iters).float().mean()), rel_v2_v1=rel(ao, bo), rel_v2_band=rel(ao[:1024], co))
print(json.dumps(out["C2"]), flush=True)
# x / y write-back parity
ax = v2.solve(cp[:2048], rpt, want_x=True, want_y=True); bx = v1.solve(cp[:2048], rpt, want_x=True, want_y=True); torch.cuda.synchronize()
out["xy"] = dict(x_maxdiff=float((ax.x - bx.x).abs().max()), y_maxdiff=float((ax.y - bx.y).abs().max()), x_scale=float(bx.x.abs().max()), y_scale=float(bx.y.abs().max()))
print(out["xy"], flush=True)
# C5 (all 560 640 LPs, cost and rhs batched)
l5, c5, w5, b5 = SC.c5()
cp5 = torch.tensor(l5, device=dev); rp5 = torch.tensor(TP.wind_battery_rparams(24, c5, w5, b5), device=dev)
a5, ms52, _ = timed(v2, cp5, rp5, reps=3); b5r, ms51, _ = timed(v1, cp5, rp5, reps=3)
out["C5"] = dict(v2_ms=ms52, v1_ms=ms51, speedup=ms51 / ms52, v2_non_optimal=int((a5.status != 0).sum()), v1_non_optimal=int((b5r.status != 0).sum()),
                 iters_v2=float(a5.iters.float().mean()), iters_max=int(a5.iters.max()), rel_v2_v1=rel(a5.obj.cpu().numpy(), b5r.obj.cpu().numpy()))
print(json.dumps(out["C5"]), flush=True)
del cp5, rp5, a5, b5r
# other horizons: every instantiation
p = SC.pool()
for T in (2, 5, 6, 7, 12, 13, 23, 24, 25, 31, 32, 33, 48, 49, 72, 96):
    tt = TP.wind_battery(T)
    s2 = S.BatchLPSolver(tt, kernel=S.KERNEL_STAGE); sb = S.BatchLPSolver(tt, kernel=S.KERNEL_BAND)
    rng = np.random.default_rng(T)
    N = 512
    starts = rng.integers(0, 8736 - T, N)
    lm = np.stack([p["dalmp_303"][s:s + T] for s in starts]) * rng.lognormal(0, 0.25, (N, T))
    cfs = np.stack([p["dacf_303"][s:s + T] for s in starts])
    rpT = TP.wind_battery_rparams(T, cfs, rng.uniform(200, 1600, N), rng.uniform(10, 800, N))
    cpd = torch.tensor(lm, device=dev); rpd = torch.tensor(rpT, device=dev)
    x2, ms, _ = timed(s2, cpd, rpd, reps=3); lg = S.last_launch(); xb, msb, _ = timed(sb, cpd, rpd, reps=3)
    out[f"T{T}"] = dict(v2_ms=ms, band_ms=msb, launch=lg, non_optimal=int((x2.status != 0).sum()), band_non_optimal=int((xb.status != 0).sum()),
                        rel=rel(x2.obj.cpu().numpy(), xb.obj.cpu().numpy()), iters=float(x2.iters.float().mean()), iters_band=float(xb.iters.float().mean()))
    print(T, json.dumps(out[f"T{T}"]), flush=True)
    s2.close(); sb.close()
json.dump(out, open("gpurun_out/stage2_check.json", "w"), indent=1)
