"""band kernel: the three placements of the per-LP work region (env DSP_BAND_MODE = smem | hybrid | ws) across templates

needs a -DDSP_PHASES build of the library, named by DSP_LP_LIB (see tools/gpu_stage2_phases.py): the product library reads no
environment, so only the instrumentation build takes DSP_BAND_MODE.  The placements are therefore compared with the phase
counters compiled in.
"""
import sys, os, json
sys.path.insert(0, ".")
import numpy as np, torch
from dispatches_b200 import templates as TP, scenarios as SC, solver as S
if not hasattr(S.load_library(), "dsp_lp_phases"):
    raise SystemExit(f"{S._LIB_PATH} is not a -DDSP_PHASES build: it ignores DSP_BAND_MODE")
dev = torch.device("cuda:0")
rng = np.random.default_rng(3)
cases = {}
cases["C4_fossil_T168"] = (TP.fossil_surrogate(168), torch.tensor(SC.c4(2000), device=dev), None)
for T, N in ((168, 2000), (96, 3000), (48, 5000)):
    cases[f"wind_battery_T{T}"] = (TP.wind_battery(T), torch.tensor(np.tile(SC.c2(N)[0], (1, T // 24)), device=dev),
                                   torch.tensor(TP.wind_battery_rparams(T, np.tile(SC.c2(1)[1], T // 24), 847.0, 211.75)[0], device=dev))
T = 48; N = 4000; cf = np.tile(SC.c2(1)[1], 2)
da = rng.uniform(5, 80, (N, T)); rt = da + rng.normal(0, 10, (N, T))
cases["bidder_da_T48"] = (TP.wind_battery_operation(T, "bidder_da"), torch.tensor(np.concatenate([da, rt, np.full((N, 1), 1e3)], 1), device=dev),
                          torch.tensor(np.repeat(TP.wind_battery_operation_rparams(T, cf, 200, 25, 100), N, 0), device=dev))
T = 24; N = 8000
sig = rng.uniform(0, 80, (N, T))
cases["tracker_T24"] = (TP.wind_battery_operation(T, "tracker"), torch.tensor(np.full((N, 1), 1e3), device=dev),
                        torch.tensor(TP.wind_battery_operation_rparams(T, np.repeat(cf[None, :T], N, 0), 200, 25, 100, 0, 0, sig), device=dev))
l2, cf2, W2, P2 = SC.c2(10000)
cases["wind_battery_pem_T24"] = (TP.wind_battery_pem(24), torch.tensor(np.concatenate([l2, np.full((10000, 1), 2.5)], axis=1), device=dev),
                                 torch.tensor(TP.wind_battery_rparams(24, cf2, W2, 150.0, pem_mw=200.0)[0], device=dev))
cases["C3_nuclear_T48"] = (TP.nuclear(48), torch.tensor(SC.c3(5000), device=dev), None)
MODES = [a.split("=")[1] for a in sys.argv if a.startswith("--modes=")]
MODES = MODES[0].split(",") if MODES else ["smem", "hybrid", "ws"]
out = {}
for name, (t, cp, rp) in cases.items():
    sol = S.BatchLPSolver(t)
    ref = None
    for mode in MODES:
        os.environ["DSP_BAND_MODE"] = mode
        o = sol.solve(cp, rp); torch.cuda.synchronize()
        ts = []
        for _ in range(2):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); sol.solve(cp, rp, out=o); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
        obj = o.obj.cpu().numpy()
        if ref is None: ref = obj
        line = dict(mode=mode, ms=min(ts), lps=cp.shape[0] / min(ts) * 1e3, nonopt=int((o.status != 0).sum()),
                    maxdiff=float((np.abs(obj - ref) / np.maximum(1, np.abs(ref))).max()), launch=S.last_launch())
        print(name, json.dumps(line)); out.setdefault(name, []).append(line)
json.dump(out, open("gpurun_out/band_modes.json", "w"), indent=1)
