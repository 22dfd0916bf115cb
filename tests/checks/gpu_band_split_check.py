"""The split band kernel (KERNEL_BAND_SPLIT) against the band kernel (KERNEL_BAND) on the same batches: kernel time from CUDA events
around the solve call after a warm-up call (best of three; the split figure includes the band kernel's retry pass behind it), iterations
(mean / max), non-optimal LPs, objective agreement, and the card's name, power limit and max SM clock.

    python tests/checks/gpu_band_split_check.py [--out DIR] [--quick]
    DSP_LP_LIB=$PWD/build/phases/libdsp_lp.so python tests/checks/gpu_band_split_check.py --counts [--out DIR]

--counts needs the -DDSP_PHASES build: it runs only the split kernel and reads the LPs whose first attempt, and whose second attempt
too, ended non-optimal (the second number is what the retry pass re-solved); it times nothing.
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np
import torch

from dispatches_b200 import scenarios as SC, solver as S, templates as TP


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def batches(quick):
    p = SC.pool()
    rng = np.random.default_rng(0)
    out = {"C4 fossil_surrogate(168) x 2000": (TP.fossil_surrogate(168), SC.c4(2000), None)}
    T = 8784
    lmp, cf = p["pq1000_rt_lmp"][:T], p["pq1000_rt_cf"][:T]
    for N in ((64,) if quick else (64, 1024)):
        h2 = rng.uniform(1.0, 3.0, N)
        cp = np.concatenate([np.tile(lmp, (N, 1)) * rng.lognormal(0, 0.1, (N, T)), h2[:, None]], axis=1)
        out[f"wind_battery_pem(8784) x {N}"] = (TP.wind_battery_pem(T), cp, TP.wind_battery_rparams(T, cf, 847.0, 150.0, pem_mw=200.0)[0])
    if not quick:
        T = 8736
        lmpd, cfd = p["pq1000_da_lmp"][:T], p["pq1000_rt_cf"][:T]
        out["wind_battery_design(8736) x 64"] = (TP.wind_battery_design(T), np.tile(lmpd, (64, 1)) * rng.lognormal(0, 0.1, (64, T)),
                                                TP.wind_battery_rparams(T, cfd, 847.0, 0.0)[0])
        T = 8784
        lam = p["nuc_report_lmp_rt"]
        reps = -(-T // len(lam))
        lamy = np.tile(lam, reps)[:T]
        cp = np.concatenate([np.tile(lamy, (64, 1)) * rng.lognormal(0, 0.1, (64, T)), rng.uniform(0.75, 3.0, (64, 1))], axis=1)
        rp = np.stack([rng.uniform(20.0, 200.0, 64), rng.uniform(0.0, 50000.0, 64), rng.uniform(0.0, 40.0, 64)], axis=1)
        out["nuclear_report(8784) x 64"] = (TP.nuclear_report(T), cp, rp)
    return out


def timed(sol, cp, rp, reps=3):
    sol.solve(cp, rp)
    torch.cuda.synchronize()
    best, r = 1e30, None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = sol.solve(cp, rp)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best, r


def counts(out_dir):
    import ctypes as C
    lib = S.load_library()
    if not hasattr(lib, "dsp_lp_phases"):
        raise SystemExit(f"{S._LIB_PATH} is not a -DDSP_PHASES build")
    buf = (C.c_ulonglong * 16)()
    dev = torch.device("cuda:0")
    rows = []
    for name, (t, cp, rp) in batches("--quick" in sys.argv).items():
        sol = S.BatchLPSolver(t, kernel=S.KERNEL_BAND_SPLIT)
        lib.dsp_lp_phases(buf, 1)
        r = sol.solve(torch.tensor(cp, device=dev), None if rp is None else torch.tensor(rp, device=dev))
        torch.cuda.synchronize()
        lib.dsp_lp_phases(buf, 1)
        row = dict(batch=name, N=len(cp), first_attempt_nonopt=int(buf[14]), both_attempts_nonopt_resolved_by_retry=int(buf[15]),
                   nonopt_after_retry=int((r.status != 0).sum().item()))
        rows.append(row)
        print(json.dumps(row))
        sol.close()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "band_split_counts.json"), "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


def main():
    out_dir = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    if "--counts" in sys.argv:
        return counts(out_dir)
    dev = torch.device("cuda:0")
    rows = []
    print("card:", card())
    for name, (t, cp, rp) in batches("--quick" in sys.argv).items():
        cpd = torch.tensor(cp, device=dev)
        rpd = None if rp is None else torch.tensor(rp, device=dev)
        res = {}
        for label, kern in (("band", S.KERNEL_BAND), ("split", S.KERNEL_BAND_SPLIT)):
            sol = S.BatchLPSolver(t, kernel=kern)
            ms, r = timed(sol, cpd, rpd)
            res[label] = dict(ms=ms, launch=S.last_launch(), obj=r.obj.cpu().numpy(), status=r.status.cpu().numpy(),
                              iters=r.iters.cpu().numpy())
            sol.close()
        b, s = res["band"], res["split"]
        ok = (s["status"] == 0) & (b["status"] == 0)
        e = np.abs(s["obj"] - b["obj"])[ok] / np.maximum(1.0, np.abs(b["obj"][ok]))
        row = dict(batch=name, m=t.m, n=t.n, w=t.w, N=len(cp), band_ms=b["ms"], split_ms=s["ms"], speedup=b["ms"] / s["ms"],
                   band_iters_mean=float(b["iters"].mean()), band_iters_max=int(b["iters"].max()),
                   split_iters_mean=float(s["iters"].mean()), split_iters_max=int(s["iters"].max()),
                   band_nonopt=int((b["status"] != 0).sum()), split_nonopt_after_retry=int((s["status"] != 0).sum()),
                   same_status=bool(np.array_equal(b["status"], s["status"])),
                   obj_rel_max=float(e.max(initial=0.0)), band_launch=b["launch"], split_launch=s["launch"])
        rows.append(row)
        print(json.dumps(row))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "band_split_check.json"), "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
