"""All 10 000 C2 LPs and the strided C5 sample (tests/real_lps.py) on the GPU through check_exact's measures: prints, per family, how
many LPs ended OPTIMAL and the largest error of every measure, and exits non-zero if any LP is not OPTIMAL or over a bar.

    python tests/checks/gpu_exact_real.py [--procs P]

Exact certification (about 7 ms per 24-hour LP on one core) and the per-LP KKT residuals run in P worker processes."""
import argparse
import multiprocessing as mp
import sys
import time
from pathlib import Path

import numpy as np

sys.path[:0] = [str(Path(__file__).resolve().parents[1]), str(Path(__file__).resolve().parents[2])]
import real_lps as R                                      # noqa: E402
from dispatches_b200 import scenarios as SC               # noqa: E402
from dispatches_b200 import solver as S                   # noqa: E402
from dispatches_b200 import templates as TP               # noqa: E402
from oracle.highs import host_cores                       # noqa: E402

_JOB = {}


def _errors(k):
    s, r = _JOB["s"], _JOB["r"]
    return R.errors(s.take(k), r.obj[k], r.x[k], r.y[k])


def _sets():
    lmp, cf, W, P = SC.c2()
    yield "C2", lmp, TP.wind_battery_rparams(24, cf, W, P)
    lmp, cf, W, P = SC.c5()
    k = np.arange(0, len(lmp), R.C5_STRIDE)
    yield "C5", lmp[k], TP.wind_battery_rparams(24, cf[k], W[k], P[k])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=host_cores())
    a = ap.parse_args()
    bad = 0
    for name, cp, rp in _sets():
        t0 = time.perf_counter()
        s = R.certify(TP.wind_battery(24), cp, rp, procs=a.procs)
        t1 = time.perf_counter()
        r = S.BatchLPSolver(s.t).solve_host(s.cparams, s.rparams, want_x=True, want_y=True)
        _JOB.update(s=s, r=r)
        chunks = np.array_split(np.arange(len(s)), 4 * a.procs)
        with mp.get_context("fork").Pool(a.procs) as pool:
            es = pool.map(_errors, chunks)
        worst = {key: max((e[key] for e in es if e[key] is not None), default=None) for key in es[0]}
        opt = int((r.status == S.OPTIMAL).sum())
        print(f"{name}: {opt} / {len(s)} OPTIMAL, {int(s.unique_x.sum())} unique in x, {int(s.unique_y.sum())} in y, "
              f"{int((s.lp_mag == 0).sum())} with a zero LP part, certified in {t1 - t0:.0f} s; largest errors {R.fmt(worst)}",
              flush=True)
        z = lambda v: 0.0 if v is None else v
        ok = (opt == len(s) and worst["obj"] <= R.OBJ_REL and z(worst["lp"]) <= R.OBJ_REL
              and max(z(worst[k]) for k in ("x", "y", "fixed", "inside")) <= R.XY_REL
              and max(worst["primal"], worst["bound"]) <= R.KKT_PRIMAL and z(worst["dual_inf"]) <= R.KKT_DUAL
              and z(worst["gap"]) <= R.KKT_GAP)
        if not ok:
            print(f"{name}: over a bar", flush=True)
            bad += 1
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
