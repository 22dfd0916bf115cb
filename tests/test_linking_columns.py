"""PV + battery + hydrogen DESIGN optimisation (size_constraints, solar_battery_hydrogen.py:205-236): the design template against the
raw oracle LP, the search for linking columns (the six scalar sizes that make A A' dense), and the numpy mirror of the bordered
normal-equation solve (oracle/ipm_border_numpy.py).  CPU only: the band kernels do not take a template with linking columns yet."""
import json
from pathlib import Path

import numpy as np
import pytest
from scipy.optimize import linprog

from dispatches_b200 import lp_template as LT, templates as TP
from oracle import highs as H, ipm_border_numpy as IB, ipm_numpy as IN, lp_models as L

GOLD = json.load(open(Path(__file__).parent / "golden" / "solar_golden.json"))
LMP = np.array(GOLD["lmp_24"])
DESIGN = GOLD["test_solar_batt_hydrogen_optimize"]
PAR = dict(pv_mw=float(DESIGN["params"]["pv_mw"]), turb_mw=float(DESIGN["params"]["turb_mw"]))


def scenarios(k):
    """scenario 0 is the reference's own case; the others perturb price, load and PV series"""
    d = L.solar_default_series()
    if k == 0:
        return LMP, d["load_mw"], d["pv_cfs"]
    rng = np.random.default_rng(100 + k)
    return LMP * rng.lognormal(0, 0.3, 24), d["load_mw"] * rng.uniform(0.7, 1.2, 24), d["pv_cfs"] * rng.uniform(0.5, 1.0, 24)


def solve_template(t, cp, rp):
    c, b, u, k = t.instantiate(cp, rp)
    r = linprog(c, A_eq=t.A, b_eq=b, bounds=[(0, None if not np.isfinite(v) else v) for v in u], method="highs-ds")
    assert r.status == 0, r.message
    return r.fun + k, r.x


@pytest.mark.parametrize("k", range(4))
def test_design_template_matches_the_raw_oracle(k):
    lmp, load, cfs = scenarios(k)
    t = TP.solar_battery_hydrogen_design(24, cfs, **PAR)
    a, x = solve_template(t, lmp, load * 1e3)
    raw = L.solar_battery_hydrogen_raw(lmp, True, PAR, pv_cfs=cfs, load_mw=load)
    b, xr = H.solve(raw)[:2]
    assert a == pytest.approx(b, rel=1e-10, abs=1e-8)
    if k == 0:                          # the reference's known answer: NPV and optimal sizes
        rep = L.solar_report(raw, xr)
        assert -a * 1e3 == pytest.approx(DESIGN["expect"]["NPV"]["value"], rel=1e-8)
        xm = x * t.col_scale + t.col_shift
        got = {nm: xm[t.column(nm)] for nm in TP.SOLAR_SIZE_COLUMNS}
        assert got["pv_add_system_capacity"] * 1e-3 == pytest.approx(DESIGN["expect"]["pv_mw"]["value"], rel=DESIGN["expect"]["pv_mw"]["rel"])
        assert got["battery_system_capacity"] * 1e-3 == pytest.approx(DESIGN["expect"]["batt_mw"]["value"], rel=DESIGN["expect"]["batt_mw"]["rel"])
        assert got["battery_system_energy"] * 1e-3 == pytest.approx(DESIGN["expect"]["batt_mwh"]["value"], rel=DESIGN["expect"]["batt_mwh"]["rel"])
        assert got["pem_system_capacity"] * 1e-3 == pytest.approx(0.0, abs=DESIGN["expect"]["pem_mw"]["abs"])
        assert got["battery_system_capacity"] == pytest.approx(rep["batt_mw"] * 1e3, rel=1e-6)


def test_linking_columns_are_the_six_sizes():
    t = TP.solar_battery_hydrogen_design(24, L.solar_default_series()["pv_cfs"], **PAR)
    assert t.w > 32                                      # A A' is dense: no band kernel takes it
    cols, perm, w = LT.find_linking_columns(t.A)
    assert sorted(t.col_names[j] for j in cols) == sorted(TP.SOLAR_SIZE_COLUMNS)
    assert w <= 32
    keep = np.setdiff1d(np.arange(t.n), cols)
    P = abs(t.A[:, keep]) @ abs(t.A[:, keep]).T
    inv = np.empty(t.m, int); inv[perm] = np.arange(t.m)
    coo = P.tocoo()
    assert np.abs(inv[coo.row] - inv[coo.col]).max() == w
    assert sorted(perm) == list(range(t.m))


@pytest.mark.parametrize("build", [lambda: TP.wind_battery(24), lambda: TP.wind_battery_design(24), lambda: TP.wind_battery_pem(24),
                                   lambda: TP.wind_battery_pem(24, with_battery=False), lambda: TP.nuclear(48),
                                   lambda: TP.fossil_surrogate(168), lambda: TP.solar_battery_hydrogen(24),
                                   lambda: TP.solar_battery_hydrogen(24, batt_mw=50.0, batt_mwh=200.0, pem_mw=20.0),
                                   lambda: TP.wind_battery_design_free_wind(24, L.solar_default_series()["pv_cfs"])])
def test_banded_templates_have_no_linking_columns(build):
    """every template that fits the band kernels today needs no linking column, and the search keeps finalize's half bandwidth"""
    t = build()
    cols, perm, w = LT.find_linking_columns(t.A)
    assert cols.size == 0 and w == t.w and w <= 32


def test_too_many_linking_columns_are_refused():
    """a dense block no handful of columns explains: no border, the full half bandwidth"""
    rng = np.random.default_rng(1)
    A = (rng.random((60, 80)) < 0.3).astype(float)
    cols, perm, w = LT.find_linking_columns(A)
    assert cols.size == 0 and w > 32


def test_dense_mirror_solves_the_design_lp():
    """the interior-point algorithm itself (dense normal equations, oracle/ipm_numpy.py) reaches the known answer on the design
    template: what a bordered band solve has to reproduce"""
    for lmp, load, cfs in map(scenarios, range(4)):
        tk = TP.solar_battery_hydrogen_design(24, cfs, **PAR)
        c, b, u, k = tk.instantiate(lmp, load * 1e3)
        r = IN.solve_batch(tk.A.toarray(), b[None], c[None], u[None])
        ref = H.solve(L.solar_battery_hydrogen_raw(lmp, True, PAR, pv_cfs=cfs, load_mw=load))[0]
        assert r["status"][0] == IN.OPTIMAL
        assert r["obj"][0] + k == pytest.approx(ref, rel=1e-8)


def _planted_border(seed, w=3, m=40, k=2, dead_rows=(), dead_scale=0.0):
    """banded A_s (half bandwidth w of A_s A_s') plus k dense columns; the entries of the rows listed in ``dead_rows`` outside the
    border are scaled by ``dead_scale`` (0: empty rows), so that M_s has a zero or tiny pivot there and the guard must catch it"""
    rng = np.random.default_rng(seed)
    cols = []
    for i in range(m):
        for _ in range(2):
            col = np.zeros(m)
            col[i] = rng.uniform(0.5, 2.0)
            j = min(m - 1, i + rng.integers(0, w + 1))
            col[j] += rng.uniform(-1.0, 1.0)
            cols.append(col)
    As = np.array(cols).T
    As[list(dead_rows)] *= dead_scale
    Ab = rng.uniform(-1.0, 1.0, (m, k))
    A = np.hstack([As, Ab])
    return A, np.arange(As.shape[1], A.shape[1])


@pytest.mark.parametrize("dead, scale", [((), 0.0), ((7,), 0.0), ((3, 21), 0.0), ((7,), 1e-7), ((3, 21), 3e-7)])
def test_guarded_bordered_solve_is_exact(dead, scale):
    """the kernel's linear algebra in the mirror: band LDL' of M_s with the pivot guard, Z = M~^-1 V, S = E^-1 + V'Z, then
    v = M~^-1 r, dy = v - Z S^-1 V'v solves the FULL normal equations -- also when rows of M_s are empty or nearly so (guarded
    pivots, q > 0; a nonzero guarded pivot p is replaced by gamma, so E carries -(gamma - p), not -gamma)"""
    A, border = _planted_border(len(dead), dead_rows=dead, dead_scale=scale)
    m, n = A.shape
    As = A.copy(); As[:, border] = 0.0
    w = max(1, max(abs(i - j) for i in range(m) for j in range(m) if (np.abs(As[i]) @ np.abs(As[j])) > 0))
    rng = np.random.default_rng(7)
    d = 10.0 ** rng.uniform(-2, 2, n)
    Mb = np.zeros((1, m + w, w + 1))
    for kk in range(w + 1):
        Mb[0, kk:m, kk] = np.einsum("ij,j,ij->i", As[kk:], d, As[:m - kk])
    guard, shift, cnt, gamma = IB._band_factor_guarded(Mb, w, 8)
    assert cnt[0] == len(dead) and sorted(guard[0, :cnt[0]]) == sorted(dead)
    assert ((shift[0, :cnt[0]] < gamma[0]) == (scale > 0)).all()
    k, q = border.size, int(cnt[0])
    V = np.zeros((1, m + w, k + q)); V[0, :m, :k] = A[:, border]
    Einv = np.concatenate([1.0 / d[border], -1.0 / shift[0, :q]])
    for g in range(q):
        V[0, guard[0, g], k + g] = 1.0
    Z = IB._band_solve(Mb, V.copy(), w)
    S = V[0, :m].T @ Z[0, :m] + np.diag(Einv)
    r = rng.standard_normal(m)
    v = np.zeros((1, m + w, 1)); v[0, :m, 0] = r
    v = IB._band_solve(Mb, v, w)[0, :m, 0]
    dy = v - Z[0, :m] @ IB._small_solve(S[None], (V[0, :m].T @ v)[None])[0]
    M = (A * d) @ A.T
    assert np.abs(M @ dy - r).max() < 1e-10 * np.abs(r).max() * np.linalg.cond(M) ** 0.5
    assert np.allclose(dy, np.linalg.solve(M, r), rtol=1e-6, atol=1e-10)



@pytest.mark.parametrize("seed", range(3))
def test_mirror_driver_without_border_is_the_dense_mirror(seed):
    """the bordered mirror's interior-point driver with no linking column (the plain band LDL') takes the iterates of
    oracle/ipm_numpy.py, iteration for iteration; a negative bound reports INFEASIBLE with NaN rows"""
    A, _ = _planted_border(seed)
    m, n = A.shape
    rng = np.random.default_rng(seed)
    u = np.full(n, 10.0)
    b = A @ rng.uniform(1.0, 9.0, n)
    c = rng.uniform(-1.0, 1.0, n)
    ref = linprog(c, A_eq=A, b_eq=b, bounds=[(0, 10.0)] * n, method="highs-ds").fun
    dense = IN.solve_batch(A, b[None], c[None], u[None])
    u2 = u.copy(); u2[3] = -1.0
    r = IB.solve_batch(A, np.stack([b, b]), np.stack([c, c]), np.stack([u, u2]), np.zeros(0, int), m - 1)
    assert r["status"][0] == IB.OPTIMAL and r["iters"][0] == dense["iters"][0]
    assert r["obj"][0] == pytest.approx(ref, rel=1e-8, abs=1e-8)
    assert r["status"][1] == IB.INFEASIBLE and np.isnan(r["obj"][1]) and np.isnan(r["x"][1]).all()


@pytest.mark.parametrize("seed", [0, 2, 6, 7, 8, 9, 10, 11, 12, 14, 15, 16])      # the seeds of range(17) whose two linking columns are basic
def test_bordered_mirror_on_planted_lps_with_basic_linking_columns(seed):
    """the mirror's interior-point driver WITH linking columns: boxed LPs (b = A x0, x0 inside the box) whose two linking columns are
    basic at HiGHS's optimum (strictly inside their bounds) end OPTIMAL within 1e-6 of HiGHS, in the dense mirror's iteration count
    +- 1"""
    A, border = _planted_border(seed)
    m, n = A.shape
    rng = np.random.default_rng(seed)
    u = np.full(n, 10.0)
    b = A @ rng.uniform(1.0, 9.0, n)
    c = rng.uniform(-1.0, 1.0, n)
    As = A.copy(); As[:, border] = 0.0
    w = max(1, max(abs(i - j) for i in range(m) for j in range(m) if (np.abs(As[i]) @ np.abs(As[j])) > 0))
    ref = linprog(c, A_eq=A, b_eq=b, bounds=[(0, 10.0)] * n, method="highs-ds")
    assert ((ref.x[border] > 1e-6) & (ref.x[border] < 10.0 - 1e-6)).all()
    r = IB.solve_batch(A, b[None], c[None], u[None], border, w)
    dense = IN.solve_batch(A, b[None], c[None], u[None])
    assert r["status"][0] == IB.OPTIMAL
    assert r["obj"][0] == pytest.approx(ref.fun, rel=1e-6, abs=1e-6)
    assert abs(int(r["iters"][0]) - int(dense["iters"][0])) <= 1
