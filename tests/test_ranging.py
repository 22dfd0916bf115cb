"""GPU tests of the ranging post-pass (dsp_lp_ranging): on every kernel family's own solve + crossover of real, degenerate dispatch LPs,
the ranges agree with the numpy mirror and, on a sample, with exact arithmetic; the kernel agrees bit for bit with its source on the SIMT
emulator and with itself in tiled batches; shared and per-LP directions; refusals, non-optimal inputs and bad bases; placement."""
import ctypes as C
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import solver as S, templates as TP  # noqa: E402
import exact_lp as E  # noqa: E402
import exact_ranging as XR  # noqa: E402
import real_lps as R  # noqa: E402
from ranging_check import against_mirror, directions, exact_checks  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

CASES = {
    "c2_stage2": (lambda: R.c2(16), {}),
    "nuclear_chain": (lambda: R.nuclear(24, N=8), {}),
    "bidder_48h_band": (lambda: R.operation("wind_battery_bidder_da", T=48, N=4), dict(kernel=S.KERNEL_BAND)),
    "fossil_band_workspace": (lambda: R.fossil(N=4), dict(kernel=S.KERNEL_BAND)),
    "fossil_band_split": (lambda: R.fossil(N=4), dict(kernel=S.KERNEL_BAND_SPLIT)),
    "design_dense": (lambda: R.solar_design(24, N=4), dict(kernel=S.KERNEL_DENSE)),
    "design_pv_dense": (lambda: R.solar_design_pv(24), dict(kernel=S.KERNEL_DENSE)),
    "tracker_band": (lambda: R.operation("wind_battery_tracker", N=4), dict(kernel=S.KERNEL_BAND)),
}
TIES_GPU = {}         # {case: [(LP, direction, side)]} near ties between the kernel's and the mirror's arithmetic

_solvers = {}


def _solver(t, kw):
    key = (id(t), tuple(sorted(kw.items())))
    if key not in _solvers:
        _solvers[key] = (t, S.BatchLPSolver(t, **kw))
    return _solvers[key][1]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")


def _host(o):
    return {f: getattr(o, f).cpu().numpy() for f in ("theta_lo", "theta_hi", "dobj", "d2obj", "status")}


def _run(s, kw, dirs=None):
    sol = _solver(s.t, kw)
    cp, rp = _dev(s.cparams), _dev(s.rparams) if s.t.Pr else None
    r = sol.solve(cp, rp, want_x=True, want_y=True)
    v = sol.crossover(cp, rp, r)
    dc, dr = (None, None) if dirs is None else (_dev(dirs[0]), _dev(dirs[1]) if s.t.Pr else None)
    g = sol.ranging(cp, rp, v, dc, dr)
    torch.cuda.synchronize()
    return sol, cp, rp, r, v, g


def _as_emu(h):
    return dict(lo=h["theta_lo"], hi=h["theta_hi"], dobj=h["dobj"], d2obj=h["d2obj"], status=h["status"])


@pytest.mark.parametrize("case", sorted(CASES))
def test_family_ranges_against_mirror_and_exact(case):
    make, kw = CASES[case]
    s = make()
    dir_c, dir_r, names = directions(s.t)
    sol, cp, rp, r, v, g = _run(s, kw, (dir_c, dir_r))
    h = _host(g)
    assert (r.status.cpu().numpy() == 0).all() and (v.status.cpu().numpy() == 0).all()
    assert (h["status"] == 0).all(), (case, h["status"])
    cs, rb = v.col_status.cpu().numpy(), v.row_basic.cpu().numpy()
    ties = against_mirror(s, (cs, rb), _as_emu(h), dir_c, dir_r, case)
    assert sorted(ties) == sorted(TIES_GPU.get(case, [])), (case, ties)
    for k in range(len(s)):                                # the first LP whose basis verifies exactly at theta = 0
        basis = (cs[k], rb[k].astype(bool))
        try:
            XR.verify(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, basis)
            break
        except E.NotCertified:
            continue
    else:
        raise AssertionError((case, "no basis of the set verifies exactly"))
    worst, checked = 0.0, 0
    for q in range(len(names)):
        if not np.isnan(h["theta_lo"][k, q]):
            worst = max(worst, exact_checks(s, k, basis, h["theta_lo"][k, q], h["theta_hi"][k, q], h["dobj"][k, q], h["d2obj"][k, q],
                                            dir_c[q], dir_r[q], (case, names[q])))
            checked += 1
    assert checked == int((~np.isnan(h["theta_lo"][k])).sum()) > 0, (case, checked)
    print(case, "theta relative error against exact", worst, "over", checked, "directions of LP", k)


@needs_gxx
@pytest.mark.parametrize("case", ["c2_stage2", "nuclear_chain", "bidder_48h_band", "design_pv_dense"])
def test_kernel_matches_its_source_on_the_emulator(case):
    import harness_ranging as H
    make, kw = CASES[case]
    s = make()
    sol, cp, rp, r, v, g = _run(s, kw)
    h = _host(g)
    e = H.run(s.t, s.cparams, s.rparams, v.status.cpu().numpy(), v.col_status.cpu().numpy(), v.row_basic.cpu().numpy())
    for a, b in (("theta_lo", "lo"), ("theta_hi", "hi"), ("dobj", "dobj"), ("d2obj", "d2obj"), ("status", "status")):
        assert np.array_equal(h[a], e[b], equal_nan=True), (case, a)


@pytest.mark.parametrize("case", ["c2_stage2", "bidder_48h_band"])
def test_tiled_batch_in_one_launch_is_bitwise_reproducible(case):
    make, kw = CASES[case]
    s = make()
    sol, cp, rp, r, v, g = _run(s, kw)
    N = len(s)
    k = np.random.default_rng(1).permutation(np.resize(np.arange(N), 3 * N + 1))
    kt = torch.as_tensor(k, device="cuda")
    vt = S.Vertex(*(getattr(v, f)[kt].contiguous() for f in ("obj", "x", "y", "col_status", "row_basic", "status", "pivots")))
    n0 = S.launch_count()
    gt = sol.ranging(cp[kt].contiguous(), rp[kt].contiguous() if rp is not None else None, vt)
    assert S.launch_count() == n0 + 1
    a, b = _host(gt), _host(g)
    for f in a:
        assert np.array_equal(a[f], b[f][k], equal_nan=True), (case, f)


def test_shared_and_per_lp_directions():
    s = R.wind_battery_pem(N=8)
    dir_c, dir_r, _ = directions(s.t)
    sol, cp, rp, r, v, g = _run(s, {}, (dir_c, dir_r))
    N = len(s)
    rng = np.random.default_rng(2)
    sc = rng.uniform(0.5, 2.0, N)                                # per LP: the shared directions scaled by a factor per LP
    pc, pr = sc[:, None, None] * dir_c[None], sc[:, None, None] * dir_r[None]
    gp = sol.ranging(cp, rp, v, _dev(pc), _dev(pr))
    a, b = _host(g), _host(gp)
    fin = np.isfinite(a["theta_hi"])
    assert np.allclose(b["theta_hi"][fin] * np.broadcast_to(sc[:, None], fin.shape)[fin], a["theta_hi"][fin], rtol=1e-12)
    assert np.array_equal(np.isinf(a["theta_hi"]), np.isinf(b["theta_hi"]))
    assert np.allclose(b["dobj"], a["dobj"] * sc[:, None], rtol=1e-12, atol=1e-12)
    one = sol.ranging(cp, rp, v, _dev(np.broadcast_to(dir_c, (N,) + dir_c.shape)), _dev(np.broadcast_to(dir_r, (N,) + dir_r.shape)))
    for f, x in _host(one).items():
        assert np.array_equal(x, a[f], equal_nan=True), f


def test_non_optimal_inputs_and_bad_bases():
    s = R.c2(8)
    sol, cp, rp, r, v, g = _run(s, {})
    cs, rb = v.col_status.clone(), v.row_basic.clone()
    st = torch.tensor([0, 1, 2, 3, 0, 0, 0, 0], dtype=torch.int32, device="cuda")
    c = cs.cpu().numpy()
    cs[4, int(np.flatnonzero(c[4] == 1)[0])] = 0                 # m - 1 members
    cs[5, int(np.flatnonzero(c[5] == 0)[0])] = 1                 # m + 1 members
    bad = S.Vertex(v.obj, v.x, v.y, cs, rb, st, v.pivots)
    h = _host(sol.ranging(cp, rp, bad))
    assert list(h["status"]) == [0, 1, 2, 3, 2, 2, 0, 0]
    no = h["status"] != 0
    for f in ("theta_lo", "theta_hi", "dobj", "d2obj"):
        assert np.isnan(h[f][no]).all() and not np.isnan(h[f][~no]).any()
    assert (h["theta_lo"][~no] <= 0).all() and (h["theta_hi"][~no] >= 0).all()


def test_refusals_and_empty_calls():
    lib = S.load_library()
    s = R.c2(2)
    sol, cp, rp, r, v, g = _run(s, {})
    K = s.t.Pc + s.t.Pr
    dc = _dev(np.eye(K, s.t.Pc))
    out = [torch.empty((2, K), dtype=torch.float64, device="cuda") for _ in range(2)] + [torch.empty(2, dtype=torch.int32, device="cuda")]
    p = lambda a: C.c_void_p(a.data_ptr()) if a is not None else None
    args = [p(v.status), p(v.col_status), p(v.row_basic), K, p(dc), None, 0, p(out[0]), p(out[1]), None, None, p(out[2]), None]
    call = lambda h, N, a, c=p(cp), rr=p(rp): lib.dsp_lp_ranging(h, N, c, rr, s.t.Pr, *a)
    assert call(None, 2, args) == -1
    assert call(sol.handle, -1, args) == -1
    for i in (0, 1, 2, 7, 8, 11):
        a = list(args); a[i] = None
        assert call(sol.handle, 2, a) == -1, i
        assert b"dsp_lp_ranging" in lib.dsp_lp_last_error()
    a = list(args); a[3] = -1
    assert call(sol.handle, 2, a) == -1 and b"K < 0" in lib.dsp_lp_last_error()
    assert call(sol.handle, 2, args, c=None) == -1 and b"cparams" in lib.dsp_lp_last_error()
    assert call(sol.handle, 2, args, rr=None) == -1 and b"rparams" in lib.dsp_lp_last_error()
    n0 = S.launch_count()
    assert call(sol.handle, 0, args) == 0 and S.launch_count() == n0
    a = list(args); a[3] = 0
    assert call(sol.handle, 2, a) == 0 and S.launch_count() == n0
    assert call(sol.handle, 2, args) == 0 and S.launch_count() == n0 + 1
    torch.cuda.synchronize()
    big = S.BatchLPSolver(TP.wind_battery(300))                   # m = 1 200
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device="cuda")
    vb = S.Vertex(z(1, torch.float64), z((1, big.t.n), torch.float64), z((1, big.t.m), torch.float64), z((1, big.t.n), torch.int8),
                  z((1, big.t.m), torch.int8), z(1, torch.int32), z(1, torch.int32))
    with pytest.raises(RuntimeError, match="m <= 1024"):
        big.ranging(_dev(np.full((1, 300), 30.0)), _dev(TP.wind_battery_rparams(300, np.full((1, 300), 0.3), 847.0, 200.0)), vb)


def test_placement_follows_m():
    _run(R.c2(4), {})
    assert S.last_launch()["smem_bytes"] > 0                    # m = 96: the work region in shared memory
    _run(R.operation("wind_battery_bidder_da", T=48, N=2), dict(kernel=S.KERNEL_BAND))
    assert S.last_launch()["smem_bytes"] == 0                   # m = 240: in the workspace
