"""The gate for linking columns in the band kernel (DESIGN §4.3), on the CPU: the bordered numpy mirror
(oracle/ipm_border_numpy.py) on the PV + battery + hydrogen design template (the reference's case + perturbed price / load series)
and on planted LPs with two basic linking columns, for several guard thresholds, against HiGHS.

    python tests/checks/border_mirror_gate.py [N_DESIGN] [EPS,EPS,...]
"""
import json
import sys

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import numpy as np
from scipy.optimize import linprog

from dispatches_b200 import lp_template as LT, templates as TP
from oracle import highs as H, ipm_border_numpy as IB, ipm_numpy as IN, lp_models as L
from test_linking_columns import _planted_border


def design(n, eps):
    lmp0 = np.array(json.load(open("tests/golden/solar_golden.json"))["lmp_24"])
    d = L.solar_default_series()
    rng = np.random.default_rng(3)
    lmp = np.vstack([lmp0[None], lmp0[None] * rng.lognormal(0, 0.3, (n - 1, 24))])
    load = np.vstack([d["load_mw"][None], d["load_mw"][None] * rng.uniform(0.7, 1.2, (n - 1, 24))])
    t = TP.solar_battery_hydrogen_design(24, d["pv_cfs"])
    cols, perm, w = LT.find_linking_columns(t.A)
    X = [t.instantiate(lmp[k], load[k] * 1e3) for k in range(n)]
    ref = np.array([H.solve(L.solar_battery_hydrogen_raw(lmp[k], True, dict(pv_mw=0.0, turb_mw=0.0), load_mw=load[k]))[0] for k in range(n)])
    A = t.A.toarray()[perm]
    out = []
    for e in eps:
        r = IB.solve_batch(A, np.array([x[1][perm] for x in X]), np.array([x[0] for x in X]), np.array([x[2] for x in X]), cols, w, eps=e)
        ok = r["status"] == IB.OPTIMAL
        err = np.abs(r["obj"] + X[0][3] - ref) / np.abs(ref)
        out.append((e, int(ok.sum()), n, float(np.nanmax(np.where(ok, err, np.nan))) if ok.any() else float("nan"), r["iters"].tolist()))
    return out


def planted(seeds, eps):
    out = []
    for e in eps:
        nopt, err, dit = 0, 0.0, []
        for seed in seeds:
            A, border = _planted_border(seed)
            m, n = A.shape
            rng = np.random.default_rng(seed)
            u = np.full(n, 10.0); b = A @ rng.uniform(1.0, 9.0, n); c = rng.uniform(-1.0, 1.0, n)
            As = A.copy(); As[:, border] = 0.0
            w = max(1, max(abs(i - j) for i in range(m) for j in range(m) if (np.abs(As[i]) @ np.abs(As[j])) > 0))
            ref = linprog(c, A_eq=A, b_eq=b, bounds=[(0, 10.0)] * n, method="highs-ds").fun
            r = IB.solve_batch(A, b[None], c[None], u[None], border, w, eps=e)
            r0 = IN.solve_batch(A, b[None], c[None], u[None])
            nopt += int(r["status"][0] == IB.OPTIMAL)
            err = max(err, abs(r["obj"][0] - ref) / max(1.0, abs(ref)))
            dit.append(int(r["iters"][0] - r0["iters"][0]))
        out.append((e, nopt, len(seeds), err, dit))
    return out


if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    eps = [float(v) for v in sys.argv[2].split(",")] if len(sys.argv) > 2 else [1e-14, 1e-12, 1e-10]
    for e, ok, tot, err, it in planted(range(16), eps):
        print(f"planted  eps={e:.0e}: {ok}/{tot} OPTIMAL, max rel err {err:.1e}, iterations minus the dense mirror's {it}")
    for e, ok, tot, err, it in design(n, eps):
        print(f"design   eps={e:.0e}: {ok}/{tot} OPTIMAL, max rel err of the optimal ones {err:.1e}, iterations {it}")
