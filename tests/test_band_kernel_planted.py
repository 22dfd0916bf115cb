"""The generic band kernel (dsp_ipm_band_kernel<W, WS, HS>) against planted-optimum LPs (tests/planted_lp.py): every padded half
bandwidth W in {1, 2, 4, 8, 16, 32} in every placement band_geometry() can produce for it, checked against the exact optimum
(objective, x and y in the caller's order), on both template set-up paths, with per-LP matrices, and through every batch /
host-staging path.

The case tables, the placements and the two (W, placement) pairs that cannot occur on an H100 are in tests/planted_lp.py.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from dispatches_b200 import solver as S
from planted_lp import AMAP_CASES, CASES, VARIANTS, band_placement, placement_of_launch, planted, shuffled
from planted_lp import rel as _rel

pytestmark = pytest.mark.gpu

N_LPS = 6
# The IPM stops at a relative duality gap below tol = 1e-9, or below 10 tol once complementarity has converged to the rounding
# floor (include/dsp_lp.h), measured on c'x of the scaled LP: a few 1e-8 were seen on an H100 (W = 32 in the workspace, 6000-LP
# batch), so the bound is 1e-7 -- still 10x inside the suite's 1e-6 against inexact references.  It applies to the whole objective
# and, separately, to the LP part c'x alone (relative to sum |c_j x*_j|), which the objective constant cannot mask.
OBJ_REL = 1e-7
XY_REL = 1e-6


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@functools.lru_cache(maxsize=None)
def _full_batch(case, amap=False):
    """the case's template with enough distinct planted LPs for more than two waves of full CTAs: several warps share a CTA's
    staged template and shared memory, and every work region is reused for later LPs"""
    kw = (AMAP_CASES if amap else CASES)[case]
    warps = band_placement(planted(seed=0, amap=amap, **kw).t)[1]
    return planted(seed=0, N=2 * _sms() * warps + 5, amap=amap, **kw), warps


def _assert_full_launch(p, pl, warps):
    ll = S.last_launch()
    assert placement_of_launch(p.t, ll) == pl, ll
    assert ll["grid"] == _sms() and ll["block"] == 32 * warps and warps > 1, (ll, warps)


def _solver(p, native):
    if native:
        t, cperm, rperm = shuffled(p.t, seed=7)
        return S.BatchLPSolver(t, native_setup=True), cperm, rperm
    return S.BatchLPSolver(p.t), None, None


def _check(p, r, cperm=None, rperm=None, what=""):
    """status, objective within OBJ_REL of the exact optimum, x / y within XY_REL of the planted ones (caller order); returns the
    largest (objective, x, y) errors"""
    assert (r.status == S.OPTIMAL).all(), (what, r.status, r.iters)
    eo = np.abs(r.obj - p.obj) / np.maximum(1.0, np.abs(p.obj))
    assert eo.max() <= OBJ_REL, (what, eo.max())
    el = np.abs(r.obj - p.obj)[p.lp_mag > 0] / p.lp_mag[p.lp_mag > 0]
    assert el.max(initial=0.0) <= OBJ_REL, (what, "LP part", el.max())
    x = p.x if cperm is None else p.x[:, cperm]
    y = p.y if rperm is None else p.y[:, rperm]
    ex = ey = 0.0
    if p.unique_x and r.x is not None:
        ex = _rel(r.x, x)
        assert ex <= XY_REL, (what, ex)
    if p.unique_y and r.y is not None:
        ey = _rel(r.y, y)
        assert ey <= XY_REL, (what, ey)
    return eo.max(), ex, ey


@pytest.mark.parametrize("native", [False, True], ids=["desc", "csr_shuffled"])
@pytest.mark.parametrize("case", sorted(CASES), ids=lambda c: f"W{c[0]}-{c[1]}")
def test_band_placement_matrix(case, native):
    W, pl = case
    p, warps = _full_batch(case)
    sol, cperm, rperm = _solver(p, native)
    m_, n_, nb_, w_ = (C.c_int32() for _ in range(4))
    assert sol.lib.dsp_lp_template_info(sol.handle, C.byref(m_), C.byref(n_), C.byref(nb_), C.byref(w_)) == 0
    assert (m_.value, n_.value, nb_.value, w_.value) == (p.t.m, p.t.n, p.t.nb, W)
    r = sol.solve_host(p.cparams, p.rparams, want_x=True, want_y=True)
    _assert_full_launch(p, pl, warps)
    _check(p, r, cperm, rperm, case)


@pytest.mark.parametrize("case", sorted(AMAP_CASES), ids=lambda c: f"W{c[0]}-{c[1]}")
def test_band_per_lp_matrix(case):
    p, warps = _full_batch(case, amap=True)
    sol, cperm, rperm = _solver(p, True)
    r = sol.solve_host(p.cparams, p.rparams, want_x=True, want_y=True)
    _assert_full_launch(p, case[1], warps)
    _check(p, r, cperm, rperm, case)


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_band_scaled_and_degenerate_data(name):
    p = planted(seed=5, N=N_LPS, **VARIANTS[name])
    for native in (False, True):
        sol, cperm, rperm = _solver(p, native)
        _check(p, sol.solve_host(p.cparams, p.rparams, want_x=True, want_y=True), cperm, rperm, (name, native))


def test_band_batches_device_and_host_paths():
    """N = 1, N below the SM count (the small-batch spread), and several waves of distinct LPs; pageable host input cut into
    chunks; the device path bitwise equal to the host path; shared and strided rparams through the C ABI"""
    p = planted(m=16, w=4, seed=11, N=6000)           # 6000 LPs: > 2 waves of 132 x 16 warps, 2 host chunks
    sol = S.BatchLPSolver(p.t)
    full = sol.solve_host(p.cparams, p.rparams, want_x=True, want_y=True)
    assert S.last_launch()["grid"] == torch.cuda.get_device_properties(0).multi_processor_count
    _check(p, full, what="N=6000")
    for N in (1, 50):
        r = sol.solve_host(p.cparams[:N], p.rparams[:N], want_x=True, want_y=True)
        ll = S.last_launch()
        assert ll["grid"] == N and (N == 1 or ll["block"] == 32), ll      # N < SMs: spread, one LP per CTA
        for a, b in ((r.obj, full.obj[:N]), (r.x, full.x[:N]), (r.y, full.y[:N]), (r.iters, full.iters[:N])):
            assert np.array_equal(a, b)
    # device tensors in / out: bitwise the host path
    dev = torch.device("cuda")
    rd = sol.solve(torch.from_numpy(p.cparams).to(dev), torch.from_numpy(p.rparams).to(dev), want_x=True, want_y=True)
    torch.cuda.synchronize()
    for a, b in ((rd.obj, full.obj), (rd.status, full.status), (rd.iters, full.iters), (rd.x, full.x), (rd.y, full.y)):
        assert np.array_equal(a.cpu().numpy(), b)
    # strided rparams rows (stride > Pr) through the C ABI
    N, Pr = 300, p.t.Pr
    rs = np.full((N, Pr + 3), np.nan); rs[:, :Pr] = p.rparams[:N]
    obj = np.empty(N); st = np.empty(N, np.int32); it = np.empty(N, np.int32); x = np.empty((N, p.t.n)); y = np.empty((N, p.t.m))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    cp = np.ascontiguousarray(p.cparams[:N])
    rc = sol.lib.dsp_lp_solve_batch_host(sol.handle, N, vp(cp), vp(rs), Pr + 3, C.byref(sol.opts), vp(obj), vp(st), vp(it), vp(x), vp(y))
    assert rc == 0
    assert np.array_equal(obj, full.obj[:N]) and np.array_equal(x, full.x[:N]) and np.array_equal(y, full.y[:N])
    # one rparams row shared by the batch
    q = planted(m=16, w=4, seed=12, N=40, shared_rparams=True)
    solq = S.BatchLPSolver(q.t)
    _check(q, solq.solve_host(q.cparams, q.rparams[0], want_x=True, want_y=True), what="shared rparams")


@pytest.mark.parametrize("native", [False, True])
def test_band_refuses_half_bandwidth_33(native):
    p = planted(m=40, w=33, seed=1)
    assert p.t.w == 33
    with pytest.raises(RuntimeError, match=r"\(-1\).*half bandwidth of A\*A' above 32"):
        S.BatchLPSolver(p.t, native_setup=native)
