"""Every kernel family's second attempt against exact optima.

Each kernel solves an LP a second time when its first attempt ends non-optimal: from the start point again, with a 0.99 step and a
10x proximal term (100x in the long-horizon and split kernels), adding the first attempt's iterations to ``iters`` and writing the
LP's rows over the first attempt's.  At default options that runs for about one LP in 1e5, so the exact-optimum suites never reach
it.  ``step_frac`` applies to the first attempt only, so a tiny one (FORCED) makes every first attempt end at the iteration cap and
every LP go through the second attempt.  Here, at the bars and with the sets, tilings and checks of the exact-optimum suites:

  a. forced retry: every LP OPTIMAL in max_iter < iters <= 2 max_iter, check_exact, every tiled copy bitwise equal to its first;
  b. restart independence: the same batch at two first-attempt step fractions that both run to the cap gives the same bits (a second
     attempt that inherits its first attempt's iterate, scaling or parked values, or a per-LP matrix modified in place, does not);
  c. mixed batches (stage 2 at every L, the chain kernel, the band kernel): at a step_frac where some LPs finish in attempt 1 and
     others need attempt 2, every LP of a tiled launch is bitwise the same LP solved alone (a slot that hands its next LP a stale
     attempt flag, iteration offset or reload mode does not);
  d. the option reaches the kernel: at step_frac 0.9 and 0.99 attempt 1 converges, passes check_exact, and differs in bits from the
     default options' result;
  e. the status rules under a forced retry: a negative bound stays INFEASIBLE (iters 0, NaN rows), a NaN price NUMERICAL, and their
     neighbours are bitwise those of a batch without them;
  f. sensitivities of retried LPs against the exact ones."""
import numpy as np
import pytest
import torch

import real_lps as R
from dispatches_b200 import solver as S
from oracle.highs import host_cores
from planted_lp import AMAP_CASES, CASES, planted
from planted_stage import CHAIN_T
from test_band_kernel_planted import OBJ_REL as BAND_OBJ_REL, _assert_full_launch, _check as _check_band, _full_batch
from test_band_kernel_planted import _solver as _band_solver
from test_band_split import PLANTED, _check_planted as _check_split, _pem_batch, _real as _split_real, _solve as _split_solve
from test_dense_exact import _run as _dense_run
from test_kernel_status_parity import BAD, _family
from test_real_lps_exact import BAND, STAGE2_T, _run, solve_device
from test_sensitivities import _exact_check as _sens_exact_check

pytestmark = pytest.mark.gpu

MAX_ITER = 60           # BatchLPSolver's default
FORCED = 1e-3           # attempt 1 cannot finish within MAX_ITER: every LP goes through attempt 2
FORCED_2 = 0.05         # nor at this step: attempt 2 must give FORCED's bits
LADDER = tuple(round(0.30 + 0.01 * k, 2) for k in range(21))      # where first-attempt and second-attempt LPs mix (test c)
MIX_SHARE = 0.1
FIELDS = ("obj", "status", "iters", "x", "y")

# What forcing the second attempt found on an H100 80GB HBM3: its parameters (step_frac 0.99, a 10x or 100x proximal term) are a design
# choice and not safer than the first attempt's on every LP.  Those LPs are pinned here, so that a change in them shows up, and every
# check runs at its full bar on the rest of their sets.
#   LPs whose second attempt ends NUMERICAL, each OPTIMAL in its first attempt at default options (set -> LP indices):
SECOND_NUMERICAL = {"band_fossil": [0], "stage2_windows96x64": [43]}
#   objective bars of the sets whose second attempt ends further from the exact objective than OBJ_REL = 1e-7 (measured largest
#   errors: 2.0e-7, 1.8e-7 and 2.0e-7 on the band kernel's planted LPs in the workspace placement, 1.04e-7 on its fossil LPs):
SECOND_OBJ_REL = {(1, "ws"): 2.5e-7, (2, "ws"): 2.5e-7, (16, "ws"): 2.5e-7, "band_fossil": 1.5e-7}
#   LPs the long and split kernels' second attempt leaves non-optimal, which the band kernel's retry pass behind them then solves at
#   the same options (set LP indices).  Of those, fossil_168 LP 0 ends NUMERICAL there too (it is band_fossil LP 0), and
#   wind_battery_pem_168 LP 3 ends 6.2e-7 from the exact objective.
LONG_LEFT = {97: [], 129: [10], 168: [10]}
SPLIT_LEFT = {"nuclear_report_96": [], "fossil_168": [0, 6], "wind_battery_pem_168": [3]}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rp(s):
    return s.rparams if s.t.Pr else None


def _assert_retried(r, what):
    """every LP OPTIMAL, attempt 1 run to its cap and attempt 2 finished"""
    assert (r.status == S.OPTIMAL).all(), (what, np.unique(r.status, return_counts=True))
    assert ((r.iters > MAX_ITER) & (r.iters <= 2 * MAX_ITER)).all(), (what, r.iters.min(), r.iters.max())


def _assert_same_bits(a, b, what, rows=None):
    for f in FIELDS:
        u, v = getattr(a, f), getattr(b, f)
        if rows is not None:
            u = u[rows]
        assert np.array_equal(u, v, equal_nan=True), (what, f)


def _restart_independent(sol2, q, r, what):
    """b: the batch q again with attempt 1 at FORCED_2 (which also runs to the cap): the same bits as r"""
    r2 = sol2.solve_host(q.cparams, _rp(q), want_x=True, want_y=True)
    assert (r2.iters > MAX_ITER).all(), (what, "attempt 1 at FORCED_2 converged", r2.iters.min())
    _assert_same_bits(r2, r, what)


def _without_numerical(s, key, solve):
    """s without the LPs SECOND_NUMERICAL[key] lists, after checking that each of them still ends NUMERICAL after both attempts under
    a forced retry and OPTIMAL at default options; solve(set, step_frac) -> LPResult"""
    bad = SECOND_NUMERICAL.get(key, [])
    if not bad:
        return s
    r = solve(s.take(bad), FORCED)
    assert (r.status == S.NUMERICAL).all() and (r.iters > MAX_ITER).all(), (key, r.status, r.iters)
    assert (solve(s.take(bad), 0.9995).status == S.OPTIMAL).all(), key
    return s.take(np.setdiff1d(np.arange(len(s)), bad))


def _host(kw):
    return lambda s, sf: S.BatchLPSolver(s.t, step_frac=sf, **kw).solve_host(s.cparams, _rp(s), want_x=True, want_y=True)


def _forced(s, name, N=None, obj_rel=R.OBJ_REL, **kw):
    """a + b for one real set on the kernel `name` runs (test_real_lps_exact._run's tiling, launch checks and check_exact)"""
    q, r = _run(s, S.BatchLPSolver(s.t, step_frac=FORCED, **kw), name, N=N, obj_rel=obj_rel)
    _assert_retried(r, name)
    _restart_independent(S.BatchLPSolver(s.t, step_frac=FORCED_2, **kw), q, r, name)
    print(name, "forced retry: iters", r.iters.min(), "..", r.iters.max())
    return q, r


# ------------------------------------------------------------------------------------------------------------------ a + b
@pytest.mark.parametrize("name", [f"T{T}" for T in STAGE2_T] + ["c2", "edges"])
def test_forced_retry_stage2(name):
    s = {"c2": lambda: R.c2(1024), "edges": R.edges}[name]() if not name[1:].isdigit() else R.windows(int(name[1:]))
    _forced(s, f"stage2_T{s.t.meta['stage_wb']['T']}")


@pytest.mark.parametrize("T", [2, 13, 24, 32])
def test_forced_retry_stage_v1(T):
    _forced(R.windows(T), "stage_v1", kernel=S.KERNEL_STAGE_V1)


@pytest.mark.parametrize("T", [97, 129, 168])
def test_forced_retry_long(T):
    """The band kernel's retry pass behind the long kernel re-solves the LPs the long kernel's second attempt leaves non-optimal: their
    rows are bitwise the band kernel's.  They must be exactly the LPs LONG_LEFT records: none at T = 97 (as in
    test_real_lps_exact.test_long), LP 10 at T = 129 and 168, whose first attempt converges at default options."""
    s = R.windows(T)
    props = torch.cuda.get_device_properties(0)
    q, r = _forced(s, "long", N=2 * _sms() * (props.max_threads_per_multi_processor // 32) + 5)
    band = S.BatchLPSolver(s.t, kernel=S.KERNEL_BAND, step_frac=FORCED).solve_host(q.cparams, q.rparams, want_x=True, want_y=True)
    _, k = s.tile(len(q), seed=1)
    left = np.unique(k[(r.x == band.x).all(1) & (r.y == band.y).all(1)])
    assert left.tolist() == LONG_LEFT[T], (T, left)


@pytest.mark.parametrize("report", [False, True], ids=["nuclear", "nuclear_report"])
@pytest.mark.parametrize("Lg", sorted(CHAIN_T))
def test_forced_retry_chain(Lg, report):
    T = CHAIN_T[Lg]
    s = R.nuclear_report(T) if report else R.nuclear(T)
    _forced(s, "chain")


@pytest.mark.parametrize("name", sorted(BAND))
def test_forced_retry_band(name):
    kw = dict(kernel=S.KERNEL_BAND)
    s = _without_numerical(BAND[name](), f"band_{name}", _host(kw))
    _forced(s, "band", obj_rel=SECOND_OBJ_REL.get(f"band_{name}", R.OBJ_REL), **kw)


def _band_planted(case, amap, native):
    p, warps = _full_batch(case, amap)
    sol, cperm, rperm = _band_solver(p, native, step_frac=FORCED)
    r = sol.solve_host(p.cparams, p.rparams, want_x=True, want_y=True)
    _assert_full_launch(p, case[1], warps)
    _assert_retried(r, case)
    _check_band(p, r, cperm, rperm, case, obj_rel=SECOND_OBJ_REL.get(case, BAND_OBJ_REL))
    sol2, _, _ = _band_solver(p, native, step_frac=FORCED_2)
    _restart_independent(sol2, p, r, case)


@pytest.mark.parametrize("native", [False, True], ids=["desc", "csr_shuffled"])
@pytest.mark.parametrize("case", sorted(CASES), ids=lambda c: f"W{c[0]}-{c[1]}")
def test_forced_retry_band_planted(case, native):
    _band_planted(case, False, native)


@pytest.mark.parametrize("native", [False, True], ids=["template_order", "csr_shuffled"])
@pytest.mark.parametrize("case", sorted(AMAP_CASES), ids=lambda c: f"W{c[0]}-{c[1]}")
def test_forced_retry_band_per_lp_matrix(case, native):
    """a per-LP matrix always takes the library's own set-up: in the template's row and column order, and shuffled"""
    _band_planted(case, True, native)


def _split_forced(t, cp, rp, what):
    """a + b on the split kernel.  The band kernel runs behind it at the same options and re-solves the LPs it leaves non-optimal,
    through the band kernel's own forced second attempt.  Returns the result and the LPs whose rows are bitwise the band kernel's at
    these options: every other row is the split kernel's own second attempt."""
    r = _split_solve(S.BatchLPSolver(t, kernel=S.KERNEL_BAND_SPLIT, step_frac=FORCED), cp, rp)
    band = S.BatchLPSolver(t, kernel=S.KERNEL_BAND, step_frac=FORCED).solve_host(cp, rp, want_x=True, want_y=True)
    left = np.flatnonzero((r.x == band.x).all(1) & (r.y == band.y).all(1))
    r2 = _split_solve(S.BatchLPSolver(t, kernel=S.KERNEL_BAND_SPLIT, step_frac=FORCED_2), cp, rp)
    assert (r2.iters > MAX_ITER).all()
    _assert_same_bits(r2, r, what)
    return r, left


@pytest.mark.parametrize("w,m", [c for c in PLANTED if c[0] in (1, 2, 4, 8)])
def test_forced_retry_split_planted(w, m):
    p = planted(m=m, w=w, seed=3, N=200)
    r, left = _split_forced(p.t, p.cparams, p.rparams, (w, m))
    assert left.size == 0, ((w, m), left)
    _assert_retried(r, (w, m))
    _check_split(p, r, what=(w, m))


@pytest.mark.parametrize("name", ["nuclear_report_96", "fossil_168", "wind_battery_pem_168"])
def test_forced_retry_split_real(name):
    s = _split_real(name)
    r, left = _split_forced(s.t, s.cparams, s.rparams, name)
    assert left.tolist() == SPLIT_LEFT[name], (name, left)
    own = np.setdiff1d(np.arange(len(s)), left)
    r = S.LPResult(*(getattr(r, f)[own] for f in FIELDS))
    _assert_retried(r, name)
    print(name, R.fmt(R.check_exact(s.take(own), r.obj, r.status, r.x, r.y, what=name)))


# the T = 24 design sets, baked and with a PV series per LP, on both dense kernels; one cluster set past 1024 rows (m = 1083, whose
# certification takes every core, as in test_dense_exact.py)
DENSE = {"solar_design24": lambda: R.solar_design(24), "solar_design_pv24": lambda: R.solar_design_pv(24),
         "solar_design72": lambda: R.solar_design(72, procs=host_cores())}


@pytest.mark.parametrize("name,kernel", [(n, k) for n in DENSE for k in ("dense", "cluster") if n.endswith("24")] +
                         [("solar_design72", "cluster")])
def test_forced_retry_dense(name, kernel):
    s = DENSE[name]()
    q, r = _dense_run(s, name, kernel, opts=dict(step_frac=FORCED))
    _assert_retried(r, (name, kernel))
    kern = {"dense": S.KERNEL_DENSE, "cluster": S.KERNEL_DENSE_CLUSTER}[kernel]
    _restart_independent(S.BatchLPSolver(s.t, kernel=kern, step_frac=FORCED_2), q, r, (name, kernel))


# ------------------------------------------------------------------------------------------------------------------ c
def _mixing_rung(sol_at, s):
    """the first step_frac of LADDER at which at least MIX_SHARE of set s finishes in attempt 1 and at least MIX_SHARE needs attempt
    2: (step_frac, LPs finished in attempt 1, LPs that ran attempt 2)"""
    seen = []
    for sf in LADDER:
        it = sol_at(sf).solve_host(s.cparams, _rp(s)).iters
        a1, a2 = int((it <= MAX_ITER).sum()), int((it > MAX_ITER).sum())
        seen.append((sf, a1, a2))
        if min(a1, a2) >= MIX_SHARE * len(it):
            return sf, a1, a2
    pytest.fail(f"no step_frac of the ladder mixes first- and second-attempt LPs (>= {MIX_SHARE:.0%} each) on this set of {len(s)} "
                f"LPs: (step_frac, attempt 1, attempt 2) = {seen}")


def _mixed(s, name, **kw):
    """c on set s: the tiled launch (test_real_lps_exact._run's size, one launch, so that group slots take second and third tickets)
    at the mixing rung, every LP bitwise the same LP solved alone; then _run's launch checks and check_exact on the same launch"""
    sol_at = lambda sf: S.BatchLPSolver(s.t, step_frac=sf, **kw)
    sf, a1, a2 = _mixing_rung(sol_at, s)
    sol = sol_at(sf)
    solve_device(sol, s.tile(40000)[0], want_xy=False)
    q, k = s.tile(2 * S.last_launch()["grid"] * S.last_launch()["problems_per_cta"] + 5, seed=1)
    r = solve_device(sol, q)
    assert (r.iters <= MAX_ITER).any() and (r.iters > MAX_ITER).any()
    for i in range(len(s)):
        solo = sol.solve_host(s.cparams[i:i + 1], _rp(s)[i:i + 1] if s.t.Pr else None, want_x=True, want_y=True)
        rows = np.flatnonzero(k == i)
        for f in FIELDS:
            a = getattr(r, f)[rows]
            assert np.array_equal(a, np.broadcast_to(getattr(solo, f), a.shape), equal_nan=True), (name, i, f)
    print(f"{name}: step_frac {sf} mixes {a1} first-attempt and {a2} second-attempt LPs of {len(s)}; {len(q)} LPs in the tiled launch, "
          "every one bitwise its solo solve")
    _run(s, sol, name, N=len(q))


@pytest.mark.parametrize("T", [5, 12, 24, 48, 96],
                         ids=lambda T: f"L{2 if T <= 6 else 4 if T <= 12 else 8 if T <= 24 else 16 if T <= 48 else 32}")
def test_mixed_batch_stage2(T):
    """64 real windows per T (63 at T = 96, without the one whose second attempt ends NUMERICAL)"""
    _mixed(_without_numerical(R.windows(T, N=64), f"stage2_windows{T}x64", _host({})), f"stage2_T{T}")


def test_mixed_batch_chain():
    _mixed(R.nuclear(48, N=64), "chain")


def test_mixed_batch_band():
    _mixed(R.c2(64), "band", kernel=S.KERNEL_BAND)


# ------------------------------------------------------------------------------------------------------------------ d
OPTION = {
    "stage2": (lambda: R.c2(64), {}),
    "stage_v1": (lambda: R.windows(24), dict(kernel=S.KERNEL_STAGE_V1)),
    "long": (lambda: R.windows(97), {}),
    "chain": (lambda: R.nuclear(48), {}),
    "band": (lambda: R.c2(64), dict(kernel=S.KERNEL_BAND)),
    "split": (lambda: _split_real("fossil_168"), dict(kernel=S.KERNEL_BAND_SPLIT)),
    "dense": (lambda: R.solar_design(24), dict(kernel=S.KERNEL_DENSE)),
    "cluster": (lambda: R.solar_design(24), dict(kernel=S.KERNEL_DENSE_CLUSTER)),
}


@pytest.mark.parametrize("family", list(OPTION))
def test_step_frac_reaches_the_kernel(family):
    mk, kw = OPTION[family]
    s = mk()
    solve = lambda **o: S.BatchLPSolver(s.t, **kw, **o).solve_host(s.cparams, _rp(s), want_x=True, want_y=True)
    default = solve()
    for sf in (0.9, 0.99):
        r = solve(step_frac=sf)
        assert (r.iters <= MAX_ITER).all(), (family, sf, r.iters.max())
        R.check_exact(s, r.obj, r.status, r.x, r.y, what=(family, sf))
        differs = (r.obj != default.obj) | (r.x != default.x).any(1) | (r.y != default.y).any(1)
        assert differs.any(), (family, sf, "bitwise the default options' result")


# ------------------------------------------------------------------------------------------------------------------ e
NAN_SLOT = 5


def _status_batch(family):
    """(template, cparams, rparams, solver kwargs, rparams column of a bound, its negative value) of test_kernel_status_parity's
    families, and of the split kernel (test_band_split's wind + battery + PEM batch) and the dense kernels on the stage-2 batch"""
    if family == "split":
        t, cp, rp = _pem_batch()
        return t, cp, rp, dict(kernel=S.KERNEL_BAND_SPLIT), 168, -5e3      # battery kW
    base = {"band": "stage2_T24", "dense": "stage2_T24", "cluster": "stage2_T24"}.get(family, family)
    t, cp, rp, kw, ib, _ = _family(base)
    kern = {"band": S.KERNEL_BAND, "dense": S.KERNEL_DENSE, "cluster": S.KERNEL_DENSE_CLUSTER}.get(family)
    if kern is not None:
        kw = dict(kw, kernel=kern)
    return t, cp, rp, kw, ib, -500.0 if base.startswith("chain") else -5e3


@pytest.mark.parametrize("family", ["stage2_T24", "stage2_T96", "stage_v1", "long_T97", "chain_report48", "band", "split", "dense",
                                    "cluster"])
def test_status_rules_under_a_forced_retry(family):
    t, cp, rp, kw, ib, neg = _status_batch(family)
    sol = S.BatchLPSolver(t, step_frac=FORCED, **kw)
    solve = (lambda c, r_: _split_solve(sol, c, r_)) if family == "split" else \
        (lambda c, r_: sol.solve_host(c, r_, want_x=True, want_y=True))
    cpb, rpb = cp.copy(), rp.copy()
    rpb[BAD, ib] = neg
    cpb[NAN_SLOT, cp.shape[1] // 2] = np.nan
    r = solve(cpb, rpb)
    assert r.status[BAD] == S.INFEASIBLE and np.isnan(r.obj[BAD]) and r.iters[BAD] == 0, (r.status[BAD], r.iters[BAD])
    assert np.isnan(r.x[BAD]).all() and np.isnan(r.y[BAD]).all()
    assert r.status[NAN_SLOT] == S.NUMERICAL, r.status[NAN_SLOT]
    keep = np.array([k for k in range(len(cp)) if k not in (BAD, NAN_SLOT)])
    ref = solve(cp[keep], rp[keep])
    _assert_retried(ref, family)
    _assert_same_bits(r, ref, family, rows=keep)


# ------------------------------------------------------------------------------------------------------------------ f
@pytest.mark.parametrize("name", ["c2", "nuclear"])
def test_sensitivities_of_retried_lps(name):
    s = {"c2": lambda: R.c2(64), "nuclear": lambda: R.nuclear(48, N=16)}[name]()
    _assert_retried(S.BatchLPSolver(s.t, step_frac=FORCED).solve_host(s.cparams, _rp(s)), name)
    print(name, _sens_exact_check(s, dict(step_frac=FORCED)))
