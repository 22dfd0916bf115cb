"""Kernel choice and chunking of the host call, one small workload per kernel family: band (every placement, the library's own setup,
per-problem matrix coefficients), band split, stage 2, long-horizon stage 2, stage v1, chain, dense (on a band template, baked, per
problem) and dense cluster.  Every workload goes through dsp_lp_solve_batch (device tensors) and dsp_lp_solve_batch_host (pageable
numpy; 4 096 LPs where the family is cheap, so that a batch the host call may cut into chunks is).  For each call the launch-count
delta, dsp_lp_last_launch and a hash of obj / status / iters go to a JSON file, so two builds of the library can be compared.  Needs a GPU.

    DSP_LP_LIB=<libdsp_lp.so> python tests/checks/host_parity.py OUT.json
"""
import hashlib
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from dispatches_b200 import scenarios as SC  # noqa: E402
from dispatches_b200 import solver as S  # noqa: E402
from dispatches_b200 import templates as TP  # noqa: E402
from oracle import lp_models as L  # noqa: E402
from planted_lp import AMAP_CASES, CASES, planted  # noqa: E402

BIG = 4096          # pageable host calls of 4 096 LPs or more are cut into chunks unless the kernel uses the handle's workspace


def _np(a):
    return a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def _digest(r):
    h = hashlib.sha256()
    for a in (r.obj, r.status, r.iters):
        h.update(np.ascontiguousarray(_np(a)).tobytes())
    return h.hexdigest()[:16]


def _run(sol, cp, rp):
    out = {}
    for how in ("solve", "solve_host"):
        if how == "solve":
            dcp = torch.from_numpy(np.ascontiguousarray(cp)).cuda()
            drp = None if rp is None else torch.from_numpy(np.ascontiguousarray(rp)).cuda()
            n0 = S.launch_count()
            r = sol.solve(dcp, drp)
            torch.cuda.synchronize()
        else:
            n0 = S.launch_count()
            r = sol.solve_host(cp, rp)
        out[how] = dict(launches=S.launch_count() - n0, last_launch=S.last_launch(), hash=_digest(r),
                        optimal=int((_np(r.status) == S.OPTIMAL).sum()), N=int(len(_np(r.obj))))
    return out


def _solar(T, N, per_problem, seed=7):
    d = L.solar_default_series()
    rng = np.random.default_rng(seed)
    lmp = 30.0 * rng.lognormal(0, 0.3, (N, T))
    load = 100.0 * rng.uniform(0.7, 1.2, (N, T))
    cf = np.tile(d["pv_cfs"], T // 24)
    reserve = np.full(T, 100.0)
    if per_problem:
        return TP.solar_battery_hydrogen_design(T, None), lmp, TP.solar_design_rparams(T, load, np.tile(cf, (N, 1)), reserve)
    return TP.solar_battery_hydrogen_design(T, cf, reserve_mw=reserve), lmp, load * 1e3


def workloads():
    for pl in ("smem_staged", "smem_l2", "hybrid", "ws"):
        p = planted(seed=1, N=BIG if pl.startswith("smem") else 512, **CASES[(4, pl)])
        yield f"band_{pl}", S.BatchLPSolver(p.t, kernel=S.KERNEL_BAND), p.cparams, p.rparams
    p = planted(seed=2, N=BIG, **CASES[(4, "smem_staged")])
    yield "band_native_setup", S.BatchLPSolver(p.t, kernel=S.KERNEL_BAND, native_setup=True), p.cparams, p.rparams
    for pl in ("smem_staged", "ws"):
        case = next(v for k, v in AMAP_CASES.items() if k[1] == pl)
        p = planted(seed=3, N=BIG if pl == "smem_staged" else 512, amap=True, **case)
        yield f"band_matrix_params_{pl}", S.BatchLPSolver(p.t, kernel=S.KERNEL_BAND), p.cparams, p.rparams
    p = planted(m=128, w=2, extra=0, bounded="none", seed=5, N=BIG)     # the band kernel of this template runs in shared memory
    yield "band_split", S.BatchLPSolver(p.t, kernel=S.KERNEL_BAND_SPLIT), p.cparams, p.rparams
    lmp, cf, W, P = SC.c2(BIG)
    rp = TP.wind_battery_rparams(24, cf, W, P)[0]
    yield "stage2", S.BatchLPSolver(TP.wind_battery(24)), lmp, rp
    yield "stage_v1", S.BatchLPSolver(TP.wind_battery(24), kernel=S.KERNEL_STAGE_V1), lmp, rp
    pool = SC.pool()
    starts = np.arange(16) * 500
    lmpl = np.stack([pool["dalmp_303"][s:s + 168] for s in starts])
    cfl = np.stack([pool["dacf_303"][s:s + 168] for s in starts])
    yield "stage2_long", S.BatchLPSolver(TP.wind_battery(168)), lmpl, TP.wind_battery_rparams(168, cfl, W, P)
    yield "chain", S.BatchLPSolver(TP.nuclear(48)), SC.c3(BIG), None
    p = planted(seed=4, N=256, m=60, w=3)
    yield "dense_on_band_template", S.BatchLPSolver(p.t, kernel=S.KERNEL_DENSE), p.cparams, p.rparams
    t, cp, rp = _solar(24, 256, False)
    yield "dense_baked", S.BatchLPSolver(t, kernel=S.KERNEL_DENSE), cp, rp
    t, cp, rp = _solar(24, 256, True)
    yield "dense_per_problem", S.BatchLPSolver(t, kernel=S.KERNEL_DENSE), cp, rp
    t, cp, rp = _solar(72, 64, False)
    yield "dense_cluster", S.BatchLPSolver(t, kernel=S.KERNEL_DENSE_CLUSTER), cp, rp


def main():
    out = sys.argv[1]
    res = {"lib": str(S._LIB_PATH)}
    for name, sol, cp, rp in workloads():
        res[name] = _run(sol, cp, rp)
        print(name, json.dumps(res[name]), flush=True)
    Path(out).parent.mkdir(parents=True, exist_ok=True)
    Path(out).write_text(json.dumps(res, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
