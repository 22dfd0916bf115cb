"""Per-LP status across the five kernel families -- stage 2 (several LPs per warp), stage v1 (lane per period), the long-horizon
stage kernel, the storage-chain kernel and the generic band kernel -- on the same LPs: negative / boundary upper bounds,
infeasible equality rows, NaN prices and the iteration cap, plus the band kernel's retry pass behind the long kernel.

The rule every kernel applies (include/dsp_lp.h): u_j < -1e-9 * beta_b is INFEASIBLE (obj NaN, iters 0, x / y rows NaN); a bound
above that is clamped to 0 and solved.  beta_b is the LP's primal scale."""
import numpy as np
import pytest

from dispatches_b200 import scenarios as SC
from dispatches_b200 import solver as S
from dispatches_b200 import templates as TP

pytestmark = pytest.mark.gpu

N = 8
BAD = 3                  # the slot that carries the bad data
SENTINEL = 12345.0


def _wb_batch(T, N=N):
    p = SC.pool()
    starts = 37 * np.arange(N) + 11
    lmp = np.stack([p["dalmp_303"][s:s + T] for s in starts])
    cf = np.stack([p["dacf_303"][s:s + T] for s in starts])
    _, _, W, P = SC.c2(1)
    return TP.wind_battery(T), lmp, TP.wind_battery_rparams(T, cf, W, P)


# family -> (template, cparams, rparams, solver kwargs, index of the bound parameter in rparams, its scale, the hour-0 rhs param)
def _family(name):
    if name.startswith("stage2") or name.startswith("long") or name == "stage_v1":
        T = int(name.split("_T")[1]) if "_T" in name else 24
        t, cp, rp = _wb_batch(T)
        kern = S.KERNEL_STAGE_V1 if name == "stage_v1" else S.KERNEL_AUTO
        return t, cp, rp, dict(kernel=kern), T, T - 1      # rparams: [wind kW * cf (T), battery kW, wind kW]
    if name == "chain_nuclear48":            # NF = 2; no rparams, so no bound can go negative
        return TP.nuclear(48), SC.c3(N), None, dict(), None, None
    if name.startswith("chain"):              # NF = 3
        t = TP.nuclear_report(48)
        lmp = SC.c3(N)
        cp = np.concatenate([lmp, np.full((N, 1), 3.0)], axis=1)
        rp = np.tile([100.0, 8000.0, 50.0], (N, 1))           # pem MW, tank kg, turbine MW
        return t, cp, rp, dict(), 1, None
    raise ValueError(name)


FAMILIES = ["stage2_T2", "stage2_T13", "stage2_T24", "stage2_T33", "stage2_T96", "stage_v1", "long_T97", "long_T128", "long_T129",
            "chain_nuclear48", "chain_report48"]
BOUNDED = [f for f in FAMILIES if f != "chain_nuclear48"]        # families whose LPs carry a bound set by rparams


def _solve(t, cp, rp, band=False, out=None, **kw):
    if band:
        kw = dict(kw, kernel=S.KERNEL_BAND)
    sol = S.BatchLPSolver(t, **kw)
    r = sol.solve_host(cp, rp, want_x=True, want_y=True, out=out)
    return r, sol


def _sentinel_out(t, n):
    return S.LPResult(np.full(n, SENTINEL), np.full(n, 7, np.int32), np.full(n, 7, np.int32), np.full((n, t.n), SENTINEL),
                      np.full((n, t.m), SENTINEL))


def _assert_rows_equal(r, ref, keep):
    """LPs `keep` of r bitwise equal to ref (which was solved without the bad LP)"""
    for a, b in ((r.obj[keep], ref.obj), (r.status[keep], ref.status), (r.iters[keep], ref.iters), (r.x[keep], ref.x), (r.y[keep], ref.y)):
        assert np.array_equal(a, b, equal_nan=True)


def _assert_kernel(name, sol):
    """the launch just made ran the family's own kernel (no silent fall-back to the band kernel)"""
    ll = S.last_launch()
    if name == "stage_v1":
        assert sol.has_stage and ll["smem_bytes"] == 0 and ll["problems_per_cta"] == ll["block"] // 32, ll   # registers only
    elif name.startswith("stage2"):
        T = int(name.split("_T")[1])
        L = 2 if T <= 6 else 4 if T <= 12 else 8 if T <= 24 else 16 if T <= 48 else 32
        assert sol.has_stage and ll["problems_per_cta"] == (32 // L) * (ll["block"] // 32), ll
    elif name.startswith("chain"):
        assert sol.has_chain1 and ll["smem_bytes"] > 0 and ll["problems_per_cta"] > ll["block"] // 32, ll
    else:                           # long horizon: the long kernel, then the band kernel's retry pass (the last launch)
        assert sol.has_stage and sol.t.meta["stage_wb"]["T"] > 96


@pytest.mark.parametrize("band", [False, True], ids=["own", "band"])
@pytest.mark.parametrize("name", BOUNDED)
def test_negative_bound(name, band):
    t, cp, rp, kw, ib, _ = _family(name)
    keep = np.array([k for k in range(N) if k != BAD])
    # a clearly negative bound: battery -5 MW / tank -500 kg
    rpb = rp.copy(); rpb[BAD, ib] = -5e3 if not name.startswith("chain") else -500.0
    r, sol = _solve(t, cp, rpb, band, out=_sentinel_out(t, N), **kw)
    if not band:
        _assert_kernel(name, sol)
    assert r.status[BAD] == S.INFEASIBLE and np.isnan(r.obj[BAD]) and r.iters[BAD] == 0
    assert np.isnan(r.x[BAD]).all() and np.isnan(r.y[BAD]).all()
    assert (r.status[keep] == S.OPTIMAL).all()
    ref, _ = _solve(t, cp[keep], rp[keep], band, **kw)
    _assert_rows_equal(r, ref, keep)


@pytest.mark.parametrize("band", [False, True], ids=["own", "band"])
@pytest.mark.parametrize("name", FAMILIES)
def test_nan_and_inf_price(name, band):
    """a NaN and an infinite price: NUMERICAL, neighbours bitwise untouched"""
    t, cp, rp, kw, _, _ = _family(name)
    keep = np.array([k for k in range(N) if k != BAD])
    ref, sol = _solve(t, cp[keep], None if rp is None else rp[keep], band, **kw)
    if not band:
        _assert_kernel(name, sol)
    for v in (np.nan, np.inf):
        cpn = cp.copy(); cpn[BAD, cp.shape[1] // 2] = v
        r, _ = _solve(t, cpn, rp, band, **kw)
        assert r.status[BAD] == S.NUMERICAL, (v, r.status[BAD])
        _assert_rows_equal(r, ref, keep)


def _boundary(name):
    """own-kernel and band-kernel status of the LP whose bound sits at -1e-13 x its scale"""
    t, cp, rp, kw, ib, icf = _family(name)
    rpb = rp.copy()
    scale = np.abs(rp[BAD, :icf + 1]).max() if icf is not None else 8000.0
    rpb[BAD, ib] = -1e-13 * scale
    own, _ = _solve(t, cp, rpb, **kw)
    band, _ = _solve(t, cp, rpb, True)
    return own.status[BAD], band.status[BAD]


@pytest.mark.parametrize("name", BOUNDED)
def test_boundary_bound_is_not_infeasible(name):
    """a bound at -1e-13 x the LP's scale is rounding, not infeasibility: every family clamps it and solves, as the band kernel does"""
    own, band = _boundary(name)
    assert own != S.INFEASIBLE and band != S.INFEASIBLE, (own, band)


# Clamping the battery bound leaves the state-of-charge row's right-hand side duration x P at -1e-13 x scale, so the clamped LP is
# infeasible by that much (include/dsp_lp.h).  Families whose elimination order handles that alike agree (OPTIMAL at T = 33 and for
# the long kernel, NUMERICAL from both at T = 2, 13, 24); where they differ the status depends on the order.
_ORDER_DEPENDENT = pytest.mark.xfail(strict=True, reason="the clamped LP is infeasible at rounding level through b = duration x P: "
                                                         "stage kernel and band kernel end with different statuses")


@pytest.mark.parametrize("name", [pytest.param(f, marks=_ORDER_DEPENDENT) if f in ("stage2_T96", "stage_v1") else f for f in BOUNDED])
def test_boundary_bound_same_status_in_every_family(name):
    own, band = _boundary(name)
    assert own == band, (own, band)


@pytest.mark.parametrize("band", [False, True], ids=["own", "band"])
@pytest.mark.parametrize("name", [f for f in FAMILIES if not f.startswith("chain")])
def test_infeasible_equality_row_is_never_optimal(name, band):
    """a negative capacity factor in one hour: g + i + q = wind * cf < 0 has no solution with g, i, q >= 0"""
    t, cp, rp, kw, ib, icf = _family(name)
    rpb = rp.copy(); rpb[BAD, 0] = -0.1 * np.abs(rp[BAD, :icf + 1]).max()
    r, _ = _solve(t, cp, rpb, band, **kw)
    assert r.status[BAD] != S.OPTIMAL


@pytest.mark.parametrize("band", [False, True], ids=["own", "band"])
@pytest.mark.parametrize("name", FAMILIES)
def test_iteration_cap_counts_both_attempts(name, band):
    t, cp, rp, kw, _, _ = _family(name)
    k = 3
    r, _ = _solve(t, cp, rp, band, max_iter=k, **kw)
    assert (r.status != S.OPTIMAL).all()
    assert (r.iters == 2 * k).all(), r.iters      # (long horizon: what the band kernel's retry pass reports, see below)


def _retry_batch():
    t, cp, rp = _wb_batch(120, N=12)
    return t, cp, rp


def test_retry_overwrites_every_lp_the_long_kernel_left():
    """with max_iter = 5 no LP converges in the long kernel, so the band kernel's retry pass re-solves all of them: AUTO gives
    bitwise the KERNEL_BAND result (a band solve is per-LP deterministic whatever the geometry)"""
    t, cp, rp = _retry_batch()
    auto, sol = _solve(t, cp, rp, max_iter=5)
    assert sol.has_stage
    band, _ = _solve(t, cp, rp, True, max_iter=5)
    for a, b in ((auto.obj, band.obj), (auto.status, band.status), (auto.iters, band.iters), (auto.x, band.x), (auto.y, band.y)):
        assert np.array_equal(a, b, equal_nan=True)


def test_retry_keeps_optimal_lps_and_infeasible_status():
    """the retry pass leaves the long kernel's OPTIMAL LPs as they are, and an INFEASIBLE LP stays INFEASIBLE with NaN rows.  (Both
    kernels apply the same bound rule and write the same NaN rows, so whether the retry skipped the INFEASIBLE LP or solved it again
    is not visible in the results.)"""
    t, cp, rp = _retry_batch()
    rpb = rp.copy(); rpb[BAD, 120] = -5e3
    auto, _ = _solve(t, cp, rpb, out=_sentinel_out(t, cp.shape[0]))
    band, _ = _solve(t, cp, rpb, True)
    assert auto.status[BAD] == S.INFEASIBLE and auto.iters[BAD] == 0 and np.isnan(auto.x[BAD]).all()
    ok = auto.status == S.OPTIMAL
    assert ok.sum() == cp.shape[0] - 1
    # the long kernel's own results stay: its elimination order rounds differently from the band kernel's
    assert not np.array_equal(auto.obj[ok], band.obj[ok])
    assert np.abs(auto.obj[ok] - band.obj[ok]).max() <= 1e-6 * np.abs(band.obj[ok]).max()
