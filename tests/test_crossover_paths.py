"""GPU tests of every path of the crossover's simplex (dsp_lp_crossover) and of the ranging over the bases it returns (dsp_lp_ranging),
on the inputs of tests/xo_lps.py: every output field, pivot counts included, is bitwise equal to the kernel's source on the SIMT
emulator -- whose path counters (tests/test_crossover_paths_cpu.py) prove which paths these inputs take -- and every OPTIMAL basis
verifies as an exact optimum.  Also: one tiled, permuted launch over every case with non-optimal inputs mixed in; planted LPs on both
sides of the shared-memory / workspace placement boundary and at m = 1024; broadcast rparams; the pivot limit; ranging against the
emulator, exact arithmetic and the numpy mirror."""
import shutil
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import solver as S  # noqa: E402
import planted_lp as PL  # noqa: E402
import xo_lps as X  # noqa: E402
from ranging_check import against_mirror, directions, exact_checks  # noqa: E402
from xo_lps import FIELDS, check_basis_exact  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

_solvers = {}
_emu = {}


def _solver(t):
    """one handle per template; the assignment LPs' A A' is dense (w > 32): the dense kernel's template"""
    if id(t) not in _solvers:
        _solvers[id(t)] = (t, S.BatchLPSolver(t, kernel=S.KERNEL_DENSE) if t.w > 32 else S.BatchLPSolver(t))
    return _solvers[id(t)][1]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")


def gpu_cross(I, max_pivots=0, rparams=None):
    """dsp_lp_crossover on the inputs (rparams: override, e.g. one broadcast row); host dict of every output field"""
    sol = _solver(I.t)
    N = len(I.x)
    rp = I.rparams if rparams is None else rparams
    r = S.LPResult(_dev(np.zeros(N)), _dev(I.status.astype(np.int32)), _dev(np.zeros(N, np.int32)), _dev(I.x), _dev(I.y))
    v = sol.crossover(_dev(I.cparams), _dev(rp) if I.t.Pr else None, r, max_pivots=max_pivots)
    torch.cuda.synchronize()
    return {f: getattr(v, f).cpu().numpy() for f in FIELDS}


def emu_cross(name):
    import harness_crossover as H
    if name not in _emu:
        I = X.ROWS[name][0]()
        _emu[name] = (I, H.run(I.t, I.cparams, I.rparams, I.status, I.x, I.y))
    return _emu[name]


def assert_same(a, b, what):
    for f in FIELDS:
        assert np.array_equal(a[f], b[f], equal_nan=True), (what, f)


@needs_gxx
@pytest.mark.parametrize("name", sorted(X.ROWS))
def test_every_case_matches_the_emulator_and_verifies_exactly(name):
    I, e = emu_cross(name)
    t0 = time.perf_counter()
    v = gpu_cross(I)
    dt = time.perf_counter() - t0
    assert_same(v, e, name)
    assert (v["status"] == X.ROWS[name][1]).all()
    for k in np.flatnonzero(v["status"] == 0):
        check_basis_exact(I, v, k)
    print(name, "largest pivot count", int(v["pivots"].max()), f"crossover call {dt * 1e3:.1f} ms")


@needs_gxx
def test_all_cases_in_one_tiled_permuted_launch():
    """every case of one template in a single launch, tiled and permuted, with LPs whose input status is not OPTIMAL mixed in: bitwise
    the emulator's outputs, and the non-optimal LPs pass through"""
    groups = {}
    for name in X.ROWS:
        I, e = emu_cross(name)
        groups.setdefault(id(I.t), []).append((I, e))
    for runs in groups.values():
        I0 = runs[0][0]
        cat = lambda f: np.concatenate([getattr(I, f) for I, _ in runs])
        ref = {f: np.concatenate([e[f] for _, e in runs]) for f in FIELDS}
        N = len(ref["obj"])
        k = np.random.default_rng(5).permutation(np.resize(np.arange(N), 2 * N + 3))
        st = np.zeros(len(k), np.int32)
        bad = np.arange(len(k)) % 4 == 1
        st[bad] = np.resize([1, 2, 3], bad.sum())
        rp = cat("rparams")[k] if I0.t.Pr else None
        n0 = S.launch_count()
        v = gpu_cross(X.Inputs(I0.t, cat("cparams")[k], rp, st, cat("x")[k], cat("y")[k]))
        assert S.launch_count() == n0 + 1
        for f in FIELDS:
            assert np.array_equal(v[f][~bad], ref[f][k][~bad], equal_nan=True), (I0.t.name, f)
        assert (v["status"][bad] == st[bad]).all() and np.isnan(v["x"][bad]).all() and np.isnan(v["obj"][bad]).all()
        assert (v["col_status"][bad] == -1).all() and (v["row_basic"][bad] == -1).all() and (v["pivots"][bad] == 0).all()


def _smem_optin():
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


@needs_gxx
def test_placement_boundary_planted():
    """planted LPs at the largest m whose work region fits in shared memory and at the next m: shared memory, then the workspace;
    both the planted optimum from a perturbed start, bitwise the emulator's"""
    import harness_crossover as H
    optin = _smem_optin()
    mb = X.planted_boundary_m(2, optin)
    for m, in_smem in ((mb, True), (mb + 1, False)):
        p = PL.planted(m, 2, N=2, extra=0, bounded="mixed", seed=m)
        assert p.t.n == 2 * m and p.t.A.nnz == X.planted_nnz(m, 2)
        assert X.in_shared_memory(m, p.t.n, p.t.A.nnz, optin) == in_smem
        I = X.planted_inputs(p, X.planted_at_u(p))
        v = gpu_cross(I)
        s = S.last_launch()["smem_bytes"]
        assert (s > 0) == in_smem, (m, s)
        if in_smem:
            assert s == X.work_doubles(m, p.t.n, p.t.A.nnz) * 8
        e = H.run(I.t, I.cparams, I.rparams, I.status, I.x, I.y)
        assert_same(v, e, m)
        for k in range(2):
            assert np.array_equal(v["col_status"][k], X.planted_basis(p, k)[0]), (m, k)
            assert np.abs(v["x"][k] - p.x[k]).max() <= 1e-12 * p.scale, (m, k)
        print("placement boundary m", m, "smem_bytes", s, "pivots", v["pivots"].tolist())


@needs_gxx
def test_assignment_past_the_boundary_crosses_over_in_the_workspace():
    import harness_crossover as H
    k = 76
    t = X.assignment_template(k)
    assert not X.in_shared_memory(t.m, t.n, t.A.nnz, _smem_optin())
    for start in ("zero", "identity"):
        I = X.assignment(k, 2, 5, start, seed=7)
        v = gpu_cross(I)
        assert S.last_launch()["smem_bytes"] == 0
        e = H.run(I.t, I.cparams, I.rparams, I.status, I.x, I.y)
        assert_same(v, e, start)
        assert (v["status"] == 0).all()
        assert np.array_equal(v["obj"], X.assignment_optimum(I.cparams.reshape(-1, k, k)))
        for q in range(2):
            check_basis_exact(I, v, q)
        print("assignment k = 76", start, "largest pivot count", int(v["pivots"].max()))


def _m1024():
    p = PL.planted(X.MAX_M, 2, N=2, extra=0, bounded="mixed", seed=11)
    assert p.t.m == X.MAX_M
    return p


def test_m1024_from_x_star_and_a_perturbed_start():
    p = _m1024()
    rng = np.random.default_rng(4)
    xp = p.x.copy()
    for k in range(2):
        col, _ = X.planted_basis(p, k)
        _, _, u, _ = p.t.instantiate(p.cparams[k], p.rparams[k])
        at0, atu, basic = col == 0, col == 2, col == 1
        span = np.where(np.isfinite(u), u, 1.0)
        xp[k, at0] = 1e-3 * span[at0] * rng.uniform(0.5, 1.0, at0.sum())
        xp[k, atu] = u[atu] - 1e-3 * u[atu] * rng.uniform(0.5, 1.0, atu.sum())
        xp[k, basic] = p.x[k, basic] * (1 + 1e-3 * rng.uniform(-1.0, 1.0, basic.sum()))
    for what, x in (("x*", p.x), ("perturbed", xp)):
        v = gpu_cross(X.planted_inputs(p, x))
        assert S.last_launch()["smem_bytes"] == 0
        assert (v["status"] == 0).all(), (what, v["status"])
        for k in range(2):
            assert np.array_equal(v["col_status"][k], X.planted_basis(p, k)[0]), (what, k)
            assert not v["row_basic"][k].any()
            assert np.abs(v["x"][k] - p.x[k]).max() <= 1e-9 * p.scale, (what, k)
            assert abs(v["obj"][k] - p.obj[k]) <= 1e-9 * max(1.0, p.lp_mag[k]), (what, k)
        print("m = 1024 from", what, "pivots", v["pivots"].tolist())


def test_m1025_is_refused():
    p = PL.planted(X.MAX_M + 1, 2, N=1, extra=0, seed=11)
    with pytest.raises(RuntimeError, match="m <= 1024"):
        gpu_cross(X.planted_inputs(p, p.x))


@needs_gxx
def test_broadcast_rparams_equal_the_rows_repeated():
    import harness_crossover as H
    p = PL.planted(40, 3, N=3, bounded="mixed", shared_rparams=True, seed=2)
    assert (p.rparams == p.rparams[0]).all()
    I = X.planted_inputs(p, X.planted_at_u(p))
    rows = gpu_cross(I)
    one = gpu_cross(I, rparams=p.rparams[0])
    assert_same(one, rows, "broadcast")
    e = H.run(I.t, I.cparams, p.rparams[0], I.status, I.x, I.y)
    assert_same(one, e, "broadcast emulator")
    assert (rows["status"] == 0).all() and (rows["pivots"] > 0).all()
    for k in range(3):
        assert np.array_equal(rows["col_status"][k], X.planted_basis(p, k)[0])


@needs_gxx
def test_pivot_limit_ends_max_iter():
    import harness_crossover as H
    I, full = emu_cross("assign40_zero_cost1000")
    one = X.Inputs(I.t, I.cparams[:1], None, I.status[:1], I.x[:1], I.y[:1])
    v = gpu_cross(one, max_pivots=1)
    assert full["pivots"][0] > 1 and v["status"][0] == 1 and v["pivots"][0] <= 1
    assert_same(v, H.run(one.t, one.cparams, None, one.status, one.x, one.y, max_pivots=1), "max_pivots=1")


# ---------------------------------------------------------------------------------------------------------------------
# ranging over the same bases
# ---------------------------------------------------------------------------------------------------------------------
RFIELDS = (("theta_lo", "lo"), ("theta_hi", "hi"), ("dobj", "dobj"), ("d2obj", "d2obj"), ("status", "status"))


def gpu_ranging(I, v, dirs=None):
    sol = _solver(I.t)
    vt = S.Vertex(*(_dev(v[f]) for f in FIELDS))
    dc, dr = (None, None) if dirs is None else (_dev(dirs[0]) if I.t.Pc else None, _dev(dirs[1]) if I.t.Pr else None)
    g = sol.ranging(_dev(I.cparams), _dev(I.rparams) if I.t.Pr else None, vt, dc, dr)
    torch.cuda.synchronize()
    return {f: getattr(g, f).cpu().numpy() for f, _ in RFIELDS}


@needs_gxx
@pytest.mark.parametrize("name", sorted(n for n in X.ROWS if X.ROWS[n][1] == 0))
def test_ranging_matches_the_emulator_on_these_bases(name):
    import harness_ranging as HR
    I, e = emu_cross(name)
    dirs = directions(I.t)[:2] if name.startswith("assign") else None       # assignment: a sample of its k^2 cost axes
    g = gpu_ranging(I, e, dirs)
    h = HR.run(I.t, I.cparams, I.rparams, e["status"], e["col_status"], e["row_basic"], *(dirs or (None, None)))
    for a, b in RFIELDS:
        assert np.array_equal(g[a], h[b], equal_nan=True), (name, a)
    assert (g["status"] == 0).all()


@needs_gxx
def test_planted_ranges_are_exact_on_every_lp_and_axis():
    """the planted bases (m = 40): every LP, every cparam and rparam axis, against exact arithmetic"""
    I, e = emu_cross("planted40_at_u")
    p = X.planted40()
    g = gpu_ranging(I, e)
    assert (g["status"] == 0).all()
    K = I.t.Pc + I.t.Pr
    dc, dr = np.eye(K, I.t.Pc), np.zeros((K, I.t.Pr))
    dr[I.t.Pc:] = np.eye(I.t.Pr)
    worst = 0.0
    for k in range(len(p.x)):
        basis = (e["col_status"][k], e["row_basic"][k].astype(bool))
        for q in range(K):
            worst = max(worst, exact_checks(p, k, basis, g["theta_lo"][k, q], g["theta_hi"][k, q], g["dobj"][k, q], g["d2obj"][k, q],
                                            dc[q], dr[q], ("planted40", k, q)))
    print("planted40 ranging: theta relative error against exact", worst, "over", len(p.x) * K, "LP-directions")


class _Batch:
    """a planted batch as ranging_check.against_mirror takes it"""
    def __init__(self, p):
        self.t, self.cparams, self.rparams = p.t, p.cparams, p.rparams

    def __len__(self):
        return len(self.cparams)


def test_m1024_ranges_against_the_mirror():
    p = _m1024()
    v = gpu_cross(X.planted_inputs(p, p.x))
    assert (v["status"] == 0).all()
    dc, dr, names = directions(p.t)
    g = gpu_ranging(X.planted_inputs(p, p.x), v, (dc, dr))
    assert (g["status"] == 0).all()
    ties = against_mirror(_Batch(p), (v["col_status"], v["row_basic"]), {b: g[a] for a, b in RFIELDS}, dc, dr, "m1024")
    assert ties == [], ties
    print("m = 1024 ranging:", len(names), "directions, finite sides", int(np.isfinite(g["theta_lo"]).sum() + np.isfinite(g["theta_hi"]).sum()))
