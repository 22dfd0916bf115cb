"""the full-year design sweep (64 LPs, T = 8736) on the stage path: long stage kernel + the band kernel's retry pass over the LPs it
left non-optimal"""
import sys
sys.path.insert(0, ".")
import numpy as np, torch
from dispatches_b200 import templates as TP, scenarios as SC, solver as S
dev = torch.device("cuda:0")
p = SC.pool()
T, N = 8736, 64
t = TP.wind_battery(T)
lam, cf = p["dalmp_303"][:T], p["dacf_303"][:T]
rng = np.random.default_rng(T)
lmp = np.tile(lam, (N, 1)) * rng.lognormal(0, 0.1, (N, T))
wind = np.repeat(np.linspace(200, 1600, 8), 8); batt = np.tile(np.linspace(0.05, 1.0, 8), 8) * wind
rp = TP.wind_battery_rparams(T, np.tile(cf, (N, 1)), wind, batt)
cpd = torch.tensor(lmp, device=dev); rpd = torch.tensor(rp, device=dev)
sol = S.BatchLPSolver(t, kernel=S.KERNEL_STAGE)
o = sol.solve(cpd, rpd); torch.cuda.synchronize()
e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
e0.record(); o = sol.solve(cpd, rpd, out=o); e1.record(); torch.cuda.synchronize()
st = o.status.cpu().numpy()
print("%.1f ms" % e0.elapsed_time(e1), "non-optimal", np.nonzero(st)[0].tolist(),
      "iters", o.iters.cpu().numpy().tolist(), "obj[19] %.10e" % float(o.obj[19]), flush=True)
