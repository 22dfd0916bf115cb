"""GPU tests of the parametric walk (dsp_lp_parametric): on every kernel family's own solve + crossover of real, degenerate dispatch LPs,
the kernel agrees bit for bit with its source on the SIMT emulator and its logs replay to bases that verify exactly; tiled and permuted
batches and per-LP directions reproduce; non-optimal inputs, empty calls and refusals; and the design identity: the minimum of the
battery-size (PEM-size) curve walked from 0 is the exact optimum of the design LP, and the design optimisation's."""
import ctypes as C
import math
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import pricetaker as PT, scenarios as SC, solver as S, templates as TP  # noqa: E402
import exact_lp as E  # noqa: E402
import exact_ranging as XR  # noqa: E402
import parametric_check as PC  # noqa: E402
import real_lps as R  # noqa: E402
from ranging_check import directions  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

CASES = {
    "c2_stage2": (lambda: R.c2(8), {}),
    "nuclear_chain": (lambda: R.nuclear(24, N=4), {}),
    "bidder_48h_band": (lambda: R.operation("wind_battery_bidder_da", T=48, N=3), dict(kernel=S.KERNEL_BAND)),
    "c4_band_workspace": (lambda: R.fossil(N=3), dict(kernel=S.KERNEL_BAND)),
    "fossil_band_split": (lambda: R.fossil(N=3), dict(kernel=S.KERNEL_BAND_SPLIT)),
    "design_dense": (lambda: R.solar_design(24, N=3), dict(kernel=S.KERNEL_DENSE)),
    "design_pv_dense": (lambda: R.solar_design_pv(24), dict(kernel=S.KERNEL_DENSE)),
}
FIELDS = ("theta", "obj", "dobj", "d2obj", "enter", "leave", "leave_to", "count", "status")
EXACT_LPS = 2
# the PV + battery + hydrogen design LPs (redundant rows, long degenerate stretches): a replayed segment basis may miss exact optimality by
# a rounding-sized primal violation (include/dsp_lp.h); there a segment's prediction is held to the exact optimum of the LP at its
# midpoint instead (parametric_check.check_walk, exact_bases=False), with the breakpoints and continuity checked as everywhere
BASES_MAY_MISS = ("design_dense", "design_pv_dense")

_solvers = {}


def _solver(t, kw):
    key = (id(t), tuple(sorted(kw.items())))
    if key not in _solvers:
        _solvers[key] = (t, S.BatchLPSolver(t, **kw))
    return _solvers[key][1]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")


def _host(o):
    return {f: getattr(o, f).cpu().numpy() for f in FIELDS}


def _run(s, kw, dirs, S_=256):
    sol = _solver(s.t, kw)
    cp, rp = _dev(s.cparams), _dev(s.rparams) if s.t.Pr else None
    r = sol.solve(cp, rp, want_x=True, want_y=True)
    v = sol.crossover(cp, rp, r)
    g = sol.parametric(cp, rp, v, _dev(dirs[0]), _dev(dirs[1]) if s.t.Pr else None, max_events=S_)
    torch.cuda.synchronize()
    return sol, cp, rp, v, g


@needs_gxx
@pytest.mark.parametrize("case", sorted(CASES))
def test_family_walks_match_the_emulator_and_verify_exactly(case):
    import harness_parametric as HP
    make, kw = CASES[case]
    s = make()
    dir_c, dir_r, names = directions(s.t, per_side=2)
    sol, cp, rp, v, g = _run(s, kw, (dir_c, dir_r))
    h = _host(g)
    vs, cs, rb = v.status.cpu().numpy(), v.col_status.cpu().numpy(), v.row_basic.cpu().numpy()
    assert (vs == 0).all()
    e = HP.run(s.t, s.cparams, s.rparams, vs, cs, rb, dir_c, dir_r if s.t.Pr else None, S=256)
    for f in FIELDS:
        assert np.array_equal(h[f], e[f], equal_nan=True), (case, f)
    moves_a = np.isnan(h["theta"][:, :, 0])
    assert (h["status"][~moves_a] != 2).all(), (case, h["status"])
    lps = checked = verified = 0
    loose = case in BASES_MAY_MISS
    for k in range(len(s)):
        basis = (cs[k], rb[k].astype(bool))
        try:
            XR.verify(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, basis)
        except E.NotCertified:
            continue
        for q in range(len(names)):
            if moves_a[k, q]:
                continue
            r = PC.check_walk(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, basis, PC.pair(h, k, q), dir_c[q],
                              dir_r[q] if s.t.Pr else None, events=False, exact_bases=not loose, what=(case, k, names[q]))
            checked += r[0] if loose else r
            verified += r[1] if loose else r
        lps += 1
        if lps == EXACT_LPS:
            break
    assert lps == EXACT_LPS and checked > 0, (case, lps, checked)
    c = h["count"][~moves_a]
    print(case, "events per walk mean", c.mean(), "max", c.max(), "segments checked exactly", checked, "of them with a basis that verifies",
          verified)


@pytest.mark.parametrize("case", ["c2_stage2", "bidder_48h_band"])
def test_tiled_permuted_batch_and_per_lp_directions_reproduce(case):
    make, kw = CASES[case]
    s = make()
    dir_c, dir_r, _ = directions(s.t, per_side=2)
    sol, cp, rp, v, g = _run(s, kw, (dir_c, dir_r))
    N = len(s)
    k = np.random.default_rng(1).permutation(np.resize(np.arange(N), 3 * N + 1))
    kt = torch.as_tensor(k, device="cuda")
    vt = S.Vertex(*(getattr(v, f)[kt].contiguous() for f in ("obj", "x", "y", "col_status", "row_basic", "status", "pivots")))
    n0 = S.launch_count()
    gt = sol.parametric(cp[kt].contiguous(), rp[kt].contiguous() if rp is not None else None, vt, _dev(dir_c), _dev(dir_r))
    assert S.launch_count() == n0 + 1
    a, b = _host(gt), _host(g)
    for f in FIELDS:
        assert np.array_equal(a[f], b[f][k], equal_nan=True), (case, f)
    gp = sol.parametric(cp, rp, v, _dev(np.broadcast_to(dir_c, (N,) + dir_c.shape)), _dev(np.broadcast_to(dir_r, (N,) + dir_r.shape)),
                        theta_end=torch.full((N, len(dir_c)), math.inf, dtype=torch.float64, device="cuda"))
    for f, x in _host(gp).items():
        assert np.array_equal(x, b[f], equal_nan=True), f


def test_non_optimal_inputs_refusals_and_empty_calls():
    lib = S.load_library()
    s = R.c2(4)
    dir_c, dir_r, _ = directions(s.t, per_side=1)
    sol, cp, rp, v, g = _run(s, {}, (dir_c, dir_r))
    st = torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda")
    bad = S.Vertex(v.obj, v.x, v.y, v.col_status, v.row_basic, st, v.pivots)
    h = _host(sol.parametric(cp, rp, bad, _dev(dir_c), _dev(dir_r)))
    assert (h["status"][1:] == np.array([1, 2, 3])[:, None]).all() and (h["count"][1:] == 0).all()
    assert np.isnan(h["theta"][1:]).all() and (h["enter"][1:] == -1).all()
    assert (h["status"][0] == 0).all() and (h["count"][0] >= 1).all()
    N, K, S_ = 4, len(dir_c), 8
    dc, dr, te = _dev(dir_c), _dev(dir_r), _dev(np.full(K, np.inf))
    f8 = lambda: torch.empty((N, K, S_), dtype=torch.float64, device="cuda")
    i4 = lambda shape: torch.empty(shape, dtype=torch.int32, device="cuda")
    outs = [f8(), f8(), f8(), f8(), i4((N, K, S_)), i4((N, K, S_)), torch.empty((N, K, S_), dtype=torch.int8, device="cuda"),
            i4((N, K)), i4((N, K))]
    p = lambda a: C.c_void_p(a.data_ptr()) if a is not None else None
    args = [p(v.status), p(v.col_status), p(v.row_basic), K, p(dc), p(dr), 0, p(te), S_] + [p(a) for a in outs]
    call = lambda h_, N_, a, c=p(cp), rr=p(rp): lib.dsp_lp_parametric(h_, N_, c, rr, s.t.Pr, *a, None)
    assert call(None, N, args) == -1
    assert call(sol.handle, -1, args) == -1
    for i in (0, 1, 2, 7, 9, 10, 11, 16, 17):                  # required pointers
        a = list(args); a[i] = None
        assert call(sol.handle, N, a) == -1, i
        assert b"dsp_lp_parametric" in lib.dsp_lp_last_error()
    a = list(args); a[8] = 0
    assert call(sol.handle, N, a) == -1 and b"S < 1" in lib.dsp_lp_last_error()
    a = list(args); a[3] = -1
    assert call(sol.handle, N, a) == -1 and b"K < 0" in lib.dsp_lp_last_error()
    for badv in (-1.0, math.nan):
        tb = te.clone(); tb[1] = badv
        a = list(args); a[7] = p(tb)
        assert call(sol.handle, N, a) == -1 and b"theta_end" in lib.dsp_lp_last_error()
    assert call(sol.handle, N, args, c=None) == -1 and b"cparams" in lib.dsp_lp_last_error()
    assert call(sol.handle, N, args, rr=None) == -1 and b"rparams" in lib.dsp_lp_last_error()
    n0 = S.launch_count()
    assert call(sol.handle, 0, args) == 0 and S.launch_count() == n0
    a = list(args); a[3] = 0
    assert call(sol.handle, N, a) == 0 and S.launch_count() == n0
    assert call(sol.handle, N, args) == 0 and S.launch_count() == n0 + 1
    torch.cuda.synchronize()
    big = S.BatchLPSolver(TP.wind_battery(300))                   # m = 1 200
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device="cuda")
    vb = S.Vertex(z(1, torch.float64), z((1, big.t.n), torch.float64), z((1, big.t.m), torch.float64), z((1, big.t.n), torch.int8),
                  z((1, big.t.m), torch.int8), z(1, torch.int32), z(1, torch.int32))
    with pytest.raises(RuntimeError, match="m <= 1024"):
        big.parametric(_dev(np.full((1, 300), 30.0)), _dev(TP.wind_battery_rparams(300, np.full((1, 300), 0.3), 847.0, 200.0)), vb,
                       _dev(np.eye(1, 300)))


def _walk_from_zero(t, cp, rp, q, kw=None):
    """solve + crossover + the walk of rparam q (1 MW = 1e3 kW) from its value in rp to +inf on the device"""
    sol = _solver(t, kw or {})
    cpd, rpd = _dev(cp), _dev(rp)
    r = sol.solve(cpd, rpd, want_x=True, want_y=True)
    v = sol.crossover(cpd, rpd, r)
    dr = np.zeros((1, t.Pr)); dr[0, q] = 1e3
    g = _host(sol.parametric(cpd, rpd, v, None, _dev(dr), max_events=512))
    return v.status.cpu().numpy(), g


def _design_identity(g, design_obj, design_mw, td, cp, rp):
    """the minimum of every convex size curve against the exact optimum of the design LP (td at cp, rp) and against the design
    optimisation's interior-point objective; the design's size lies in the arg-min stretch.  Returns the worst relative errors
    (exact, interior point) and the number of LPs certified exactly."""
    worst_x = worst_i = 0.0
    certified = 0
    for k in range(len(design_obj)):
        c = int(g["count"][k, 0])
        assert g["status"][k, 0] == 0, (k, g["status"][k, 0])
        ob, th = g["obj"][k, 0, :c], g["theta"][k, 0, :c]
        e = int(np.argmin(ob))
        try:
            ex = E.exact_optimum(td, cp[k], rp[k]).obj
            worst_x = max(worst_x, abs(ob[e] - ex) / max(1.0, abs(ex)))
            certified += 1
        except E.NotCertified:
            pass
        worst_i = max(worst_i, abs(ob[e] - design_obj[k]) / max(1.0, abs(design_obj[k])))
        lo = th[e - 1] if e > 0 else 0.0                            # the flat stretch around the minimum
        hi = th[e + 1] if e + 1 < c else math.inf
        flat = np.flatnonzero(np.abs(ob - ob[e]) <= 1e-9 * max(1.0, abs(ob[e])))
        lo, hi = min(lo, th[flat].min()), max(hi, th[flat].max() if flat.max() + 1 >= c else th[flat.max() + 1])
        assert lo - 1e-6 * max(1.0, hi) <= design_mw[k] <= hi + 1e-6 * max(1.0, hi), (k, design_mw[k], lo, hi)
    return worst_x, worst_i, certified


@pytest.mark.parametrize("T,N", [(24, 256), (48, 64)])
def test_battery_size_curve_minimum_is_the_design_optimum(T, N):
    lmp, cf, W, _ = SC.c2(N, seed=11) if T == 24 else (None, None, None, None)
    if T != 24:
        p = SC.pool()
        h0 = np.random.default_rng(3).integers(0, len(p["dalmp_303"]) - T, N)
        idx = h0[:, None] + np.arange(T)[None, :]
        lmp, cf, W = p["dalmp_303"][idx], p["dacf_303"][idx], SC.FIXED_WIND_MW
    cf = np.broadcast_to(np.asarray(cf, float)[..., :T], (N, T))
    t = TP.wind_battery(T)
    rp = TP.wind_battery_rparams(T, cf, W, 0.0)
    vs, g = _walk_from_zero(t, lmp, rp, T)
    assert (vs == 0).all()
    d = PT.wind_battery_optimize(T, dict(DA_LMPs=lmp, wind_resource=cf, wind_mw=W, batt_mw=0.0, design_opt=True))
    assert (d.status == 0).all()
    wx, wi, cert = _design_identity(g, d.obj, d.sizes["batt_kw"] / 1e3, TP.wind_battery_design(T), lmp, rp)
    print(f"T = {T}: {N} battery-size curves; minimum against the exact design optimum (certified {cert}): worst relative error "
          f"{wx:.2e}, against the interior-point design solve {wi:.2e}; events mean {g['count'].mean():.1f} max {g['count'].max()}")
    assert cert >= N // 2 and wx <= 1e-9 and wi <= 1e-7


def test_pem_size_curve_minimum_is_the_pem_design_optimum():
    T, N = 24, 64
    lmp, cf, W, _ = SC.c2(N, seed=5)
    cf = np.broadcast_to(np.asarray(cf, float)[..., :T], (N, T))
    t = TP.wind_battery_pem(T, with_battery=False)
    cp = np.concatenate([lmp, np.full((N, 1), 2.5)], axis=1)
    rp = TP.wind_battery_rparams(T, cf, W, 0.0, pem_mw=0.0)
    vs, g = _walk_from_zero(t, cp, rp, T + 2)
    assert (vs == 0).all()
    d = PT.wind_battery_pem_optimize(T, dict(DA_LMPs=lmp, wind_resource=cf, wind_mw=W, batt_mw=0.0, pem_mw=0.0, h2_price_per_kg=2.5,
                                             design_opt="PEM"))
    assert (d.status == 0).all()
    wx, wi, cert = _design_identity(g, d.obj, d.sizes["pem_kw"] / 1e3, TP.wind_battery_pem(T, with_battery=False, pem_design=True), cp,
                                    rp)
    print(f"{N} PEM-size curves; minimum against the exact PEM design optimum (certified {cert}): worst relative error {wx:.2e}, "
          f"against the interior-point design solve {wi:.2e}")
    assert cert >= N // 2 and wx <= 1e-9 and wi <= 1e-7
