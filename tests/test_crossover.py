"""GPU tests of the crossover post-pass (dsp_lp_crossover): on each kernel family's own (x, y) of real, degenerate dispatch LPs, every
basis the kernel returns verifies as an exact optimum (exact_lp.exact_optimum with basis=); tiled batches are bitwise reproducible; the
kernel agrees bit for bit with its source on the SIMT emulator started from the same (x, y); refusals and non-optimal inputs."""
import ctypes as C
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import solver as S, templates as TP  # noqa: E402
import real_lps as R  # noqa: E402
from crossover_check import check_vertices  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

# (set, kernel family): how the set is solved before the crossover
CASES = {
    "c2_stage2": (lambda: R.c2(32), {}),
    "edges_stage2": (lambda: R.edges(), {}),
    "nuclear_chain": (lambda: R.nuclear(24), {}),
    "fossil_band_workspace": (lambda: R.fossil(), dict(kernel=S.KERNEL_BAND)),
    "fossil_band_split": (lambda: R.fossil(), dict(kernel=S.KERNEL_BAND_SPLIT)),
    "design_dense": (lambda: R.solar_design(24), dict(kernel=S.KERNEL_DENSE)),
    "design_pv_dense": (lambda: R.solar_design_pv(24), dict(kernel=S.KERNEL_DENSE)),
    "design_dense_cluster": (lambda: R.solar_design(24), dict(kernel=S.KERNEL_DENSE_CLUSTER)),
    "c2_dense_cluster": (lambda: R.c2(16), dict(kernel=S.KERNEL_DENSE_CLUSTER)),
}
CASES.update({f"{name}_band": ((lambda name=name: R.operation(name)), dict(kernel=S.KERNEL_BAND)) for name in R.OPERATIONS})
CASES["bidder_48h_band"] = (lambda: R.operation("wind_battery_bidder_da", T=48), dict(kernel=S.KERNEL_BAND))

# LPs whose GPU basis is primal infeasible in exact arithmetic by rounding, certified after exact_lp._repair with these pivots
PINNED_GPU = {}

_solvers = {}


def _solver(t, kw):
    key = (id(t), tuple(sorted(kw.items())))
    if key not in _solvers:
        _solvers[key] = (t, S.BatchLPSolver(t, **kw))
    return _solvers[key][1]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")


def _solve_and_cross(s, kw, tile=None):
    sol = _solver(s.t, kw)
    cp, rp = _dev(s.cparams), _dev(s.rparams) if s.t.Pr else None
    r = sol.solve(cp, rp, want_x=True, want_y=True)
    v = sol.crossover(cp, rp, r)
    torch.cuda.synchronize()
    host = lambda o: {f: getattr(o, f).cpu().numpy() for f in ("obj", "x", "y", "col_status", "row_basic", "status", "pivots")}
    return sol, r, host(v)


@pytest.mark.parametrize("case", sorted(CASES))
def test_family_vertices_are_exact_optima(case):
    make, kw = CASES[case]
    s = make()
    sol, r, v = _solve_and_cross(s, kw)
    status = r.status.cpu().numpy()
    assert (status == 0).all(), (case, status)
    piv = check_vertices(s, v, status, PINNED_GPU.get(case), case)
    print(case, "pivots max", int(piv.max()), "mean", float(piv.mean()))


@needs_gxx
@pytest.mark.parametrize("case", ["c2_stage2", "nuclear_chain", "wind_battery_bidder_da_band", "design_pv_dense"])
def test_kernel_matches_its_source_on_the_emulator(case):
    import harness_crossover as H
    make, kw = CASES[case]
    s = make()
    sol, r, v = _solve_and_cross(s, kw)
    e = H.run(s.t, s.cparams, s.rparams, r.status.cpu().numpy(), r.x.cpu().numpy(), r.y.cpu().numpy())
    for f in ("obj", "x", "y", "col_status", "row_basic", "status", "pivots"):
        assert np.array_equal(v[f], e[f], equal_nan=True), (case, f)


@pytest.mark.parametrize("case", ["c2_stage2", "wind_battery_tracker_band", "fossil_band_workspace"])
def test_tiled_batch_is_bitwise_reproducible(case):
    make, kw = CASES[case]
    s = make()
    sol = _solver(s.t, kw)
    cp, rp = _dev(s.cparams), _dev(s.rparams) if s.t.Pr else None
    r = sol.solve(cp, rp, want_x=True, want_y=True)
    N = len(s)
    k = np.random.default_rng(1).permutation(np.resize(np.arange(N), 3 * N + 1))
    kt = torch.as_tensor(k, device="cuda")
    rt = S.LPResult(r.obj[kt].contiguous(), r.status[kt].contiguous(), r.iters[kt].contiguous(), r.x[kt].contiguous(), r.y[kt].contiguous())
    n0 = S.launch_count()
    vt = sol.crossover(cp[kt].contiguous(), rp[kt].contiguous() if rp is not None else None, rt)
    assert S.launch_count() == n0 + 1
    v = sol.crossover(cp, rp, r)
    torch.cuda.synchronize()
    for f in ("obj", "x", "y", "col_status", "row_basic", "status", "pivots"):
        a, b = getattr(vt, f).cpu().numpy(), getattr(v, f).cpu().numpy()
        assert np.array_equal(a, b[k], equal_nan=True), (case, f)
    one = sol.crossover(cp[:1].contiguous(), rp[:1].contiguous() if rp is not None else None,
                        S.LPResult(r.obj[:1], r.status[:1], r.iters[:1], r.x[:1].contiguous(), r.y[:1].contiguous()))
    assert np.array_equal(one.x.cpu().numpy()[0], v.x.cpu().numpy()[0])
    assert np.array_equal(one.col_status.cpu().numpy()[0], v.col_status.cpu().numpy()[0])


def test_placement_follows_m():
    s = R.c2(4)
    _solve_and_cross(s, {})
    assert S.last_launch()["smem_bytes"] > 0                 # m = 96: B^-1 in shared memory
    s = R.operation("wind_battery_bidder_da", T=48)
    _solve_and_cross(s, dict(kernel=S.KERNEL_BAND))
    assert S.last_launch()["smem_bytes"] == 0                # m = 240: B^-1 in the workspace


def test_non_optimal_inputs_pass_through():
    s = R.c2(6)
    sol, r, _ = _solve_and_cross(s, {})
    st = torch.tensor([0, 1, 2, 3, 0, 1], dtype=torch.int32, device="cuda")
    r2 = S.LPResult(r.obj, st, r.iters, r.x, r.y)
    v = sol.crossover(_dev(s.cparams), _dev(s.rparams), r2)
    st = st.cpu().numpy(); bad = st != 0
    vs = v.status.cpu().numpy()
    assert (vs[bad] == st[bad]).all() and (vs[~bad] == 0).all()
    assert np.isnan(v.x.cpu().numpy()[bad]).all() and np.isnan(v.y.cpu().numpy()[bad]).all() and np.isnan(v.obj.cpu().numpy()[bad]).all()
    assert (v.col_status.cpu().numpy()[bad] == -1).all() and (v.row_basic.cpu().numpy()[bad] == -1).all()
    assert (v.pivots.cpu().numpy()[bad] == 0).all()


def test_refusals_and_empty_batch():
    lib = S.load_library()
    s = R.c2(2)
    sol, r, _ = _solve_and_cross(s, {})
    cp, rp = _dev(s.cparams), _dev(s.rparams)
    out = [torch.empty(2, dtype=torch.float64, device="cuda"), torch.empty((2, s.t.n), dtype=torch.float64, device="cuda"),
           torch.empty((2, s.t.m), dtype=torch.float64, device="cuda"), torch.empty(2, dtype=torch.int32, device="cuda")]
    p = lambda a: C.c_void_p(a.data_ptr()) if a is not None else None
    call = lambda h, N, st, x, y, obj, xo, yo, xs: lib.dsp_lp_crossover(h, N, p(cp), p(rp), s.t.Pr, st, x, y, 0, obj, xo, yo, None, None,
                                                                          xs, None, None)
    good = (p(r.status), p(r.x), p(r.y), p(out[0]), p(out[1]), p(out[2]), p(out[3]))
    assert call(None, 2, *good) == -1
    assert call(sol.handle, -1, *good) == -1
    for k in range(7):
        args = list(good); args[k] = None
        assert call(sol.handle, 2, *args) == -1
        assert b"dsp_lp_crossover" in lib.dsp_lp_last_error()
    # missing parameter arrays: the template has Pc = 24 and Pr = 26
    assert lib.dsp_lp_crossover(sol.handle, 2, None, p(rp), s.t.Pr, *good[:3], 0, *good[3:6], None, None, good[6], None, None) == -1
    assert b"cparams" in lib.dsp_lp_last_error()
    assert lib.dsp_lp_crossover(sol.handle, 2, p(cp), None, s.t.Pr, *good[:3], 0, *good[3:6], None, None, good[6], None, None) == -1
    assert b"rparams" in lib.dsp_lp_last_error()
    n0 = S.launch_count()
    assert call(sol.handle, 0, *good) == 0 and S.launch_count() == n0
    assert call(sol.handle, 2, *good) == 0 and S.launch_count() == n0 + 1
    torch.cuda.synchronize()
    big = S.BatchLPSolver(TP.wind_battery(300))                   # m = 1 200
    with pytest.raises(RuntimeError, match="m <= 1024"):
        lmp = _dev(np.full((1, 300), 30.0))
        rpb = _dev(TP.wind_battery_rparams(300, np.full((1, 300), 0.3), 847.0, 200.0))
        rb = S.LPResult(torch.zeros(1, dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
                        torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros((1, big.t.n), dtype=torch.float64, device="cuda"),
                        torch.zeros((1, big.t.m), dtype=torch.float64, device="cuda"))
        big.crossover(lmp, rpb, rb)


def test_sensitivities_accept_the_vertex():
    s = R.nuclear(24)
    sol, r, _ = _solve_and_cross(s, {})
    cp = _dev(s.cparams)
    v = sol.crossover(cp, None, r)
    at_v = sol.sensitivities(cp, None, S.LPResult(v.obj, v.status, r.iters, v.x, v.y))
    at_i = sol.sensitivities(cp, None, r)
    torch.cuda.synchronize()
    rc, cs = at_v.rc.cpu().numpy(), v.col_status.cpu().numpy()
    sd = np.abs(s.cparams).max(1, keepdims=True)
    assert (v.status.cpu().numpy() == 0).all() and np.isfinite(rc).all()
    assert (np.abs(rc[cs == 1]) <= 1e-9 * np.broadcast_to(sd, rc.shape)[cs == 1]).all()      # basic columns: zero reduced cost
    assert (rc[cs == 0] >= -1e-9 * np.broadcast_to(sd, rc.shape)[cs == 0]).all()
    assert (rc[cs == 2] <= 1e-9 * np.broadcast_to(sd, rc.shape)[cs == 2]).all()
    # where y* is unique, the interior point's duals agree with the vertex's basis duals to the interior-point method's own accuracy
    uy = s.unique_y
    if uy.any():
        dv, di = at_v.d_cparams.cpu().numpy()[uy], at_i.d_cparams.cpu().numpy()[uy]
        assert (np.abs(dv - di) / np.maximum(1.0, np.abs(dv).max(1, keepdims=True))).max() <= 1e-6


@pytest.mark.parametrize("case", ["c2_stage2", "nuclear_chain", "wind_battery_bidder_da_band", "design_dense"])
def test_gpu_basis_against_the_numpy_mirror(case):
    """the numpy mirror (oracle/crossover_numpy.py) started from the GPU's x: its basis verifies exactly, and where it differs from
    the kernel's (a near tie met with different arithmetic) both are exact optima; the LPs that differ are reported"""
    import exact_lp as E
    from oracle import crossover_numpy as XN
    make, kw = CASES[case]
    s = make()
    sol, r, v = _solve_and_cross(s, kw)
    x = r.x.cpu().numpy()
    from crossover_check import _repair_pivots
    differ, repaired = [], {}
    for k in range(len(s)):
        c, b, u, _ = s.t.instantiate(s.cparams[k], s.rparams[k])
        mr = XN.crossover(s.t.matrix(s.rparams[k]), b, c, u, x[k])
        assert mr["status"] == 0
        basis = (mr["col_status"], mr["row_basic"].astype(bool))
        try:
            E.exact_optimum(s.t, s.cparams[k], s.rparams[k], basis=basis)
        except E.NotCertified:
            # the mirror solves without refinement: a degenerate basic variable can come out exactly infeasible by rounding, as
            # HiGHS' bases on these LPs do; it is certified after exact_lp._repair
            repaired[k] = _repair_pivots(s, k, basis)
        if not (np.array_equal(mr["col_status"], v["col_status"][k]) and np.array_equal(mr["row_basic"], v["row_basic"][k])):
            differ.append(k)
    print(case, "LPs where the mirror's basis differs from the GPU's (both verified):", differ, "mirror bases repaired:", repaired)
    if case != "design_dense":       # the design LPs take about 130 degenerate pivots each: the two paths part at a near tie on most
        assert len(differ) <= len(s) // 2, differ
    assert max(repaired.values(), default=0) <= 8, repaired
