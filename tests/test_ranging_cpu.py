"""CPU tests of the ranging post-pass (dsp_lp_ranging): the CTA body of dispatches_b200/csrc/dsp_ranging.cuh on the SIMT emulator, on the
bases the emulated crossover returns from the numpy interior-point mirrors' (x, y) on real, degenerate dispatch LPs; against the numpy
mirror (oracle/ranging_numpy.py), against exact arithmetic (exact_ranging) and against the sensitivity pass's gradient."""
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

from dispatches_b200 import scenarios as SC, templates as TP  # noqa: E402
import exact_lp as E  # noqa: E402
import exact_ranging as XR  # noqa: E402
import real_lps as R  # noqa: E402
from crossover_check import interior_xy  # noqa: E402
from ranging_check import against_mirror, directions, exact_checks  # noqa: E402

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

SETS = {
    "c2": (lambda: R.c2(8), False),
    "nuclear": (lambda: R.nuclear(24, N=8), False),
    "wind_battery_pem": (lambda: R.wind_battery_pem(N=8), False),
    "design": (lambda: R.design(24, N=4), True),
    "solar_design": (lambda: R.solar_design(24, N=4), True),
    "solar_design_pv": (lambda: R.solar_design_pv(24), True),
    "fossil": (lambda: R.fossil(N=4), False),
}
SETS.update({f"operation_{name}": ((lambda name=name: R.operation(name, N=4)), False) for name in R.OPERATIONS})

# (set, LP, direction index) where a ratio test meets a near tie between the kernel's and the mirror's arithmetic
TIES = {}
EXACT_SAMPLE = 2          # LPs per set checked in exact arithmetic

_cache = {}


def _bases(name):
    """(set, emulated crossover output) of a set, cached"""
    if name not in _cache:
        import harness_crossover as HX
        make, dense = SETS[name]
        s = make()
        status, x, y = interior_xy(s, dense)
        _cache[name] = (s, HX.run(s.t, s.cparams, s.rparams, status, x, y))
    return _cache[name]


def _ranging(s, v, dir_c, dir_r):
    import harness_ranging as H
    return H.run(s.t, s.cparams, s.rparams, v["status"], v["col_status"], v["row_basic"], dir_c, dir_r)


@needs_gxx
@pytest.mark.parametrize("name", sorted(SETS))
def test_emulated_kernel_against_mirror_and_exact(name):
    s, v = _bases(name)
    assert (v["status"] == 0).all(), (name, v["status"])
    dir_c, dir_r, names = directions(s.t)
    out = _ranging(s, v, dir_c, dir_r)
    assert (out["status"] == 0).all(), (name, out["status"])
    ties = against_mirror(s, (v["col_status"], v["row_basic"]), out, dir_c, dir_r, name)
    assert sorted(ties) == sorted(TIES.get(name, [])), (name, ties)
    worst, checked, lps = 0.0, 0, 0
    for k in range(len(s)):
        if lps == EXACT_SAMPLE:
            break
        basis = (v["col_status"][k], v["row_basic"][k].astype(bool))
        try:
            XR.verify(s.t, s.cparams[k], s.rparams[k] if s.t.Pr else None, basis)
        except E.NotCertified:
            continue                                       # only bases that verify exactly at theta = 0 are ranged exactly
        lps += 1
        for q in range(len(names)):
            if np.isnan(out["lo"][k, q]):
                continue
            worst = max(worst, exact_checks(s, k, basis, out["lo"][k, q], out["hi"][k, q], out["dobj"][k, q], out["d2obj"][k, q],
                                            dir_c[q], dir_r[q], (name, names[q])))
            checked += 1
    # EXACT_SAMPLE LPs of every set, every direction that does not move A, went through the exact checks
    assert lps == EXACT_SAMPLE and checked == EXACT_SAMPLE * int((~np.isnan(out["lo"][0])).sum()), (name, lps, checked)
    print(name, "theta relative error against exact", worst, "over", checked, "(LP, direction) pairs")


@needs_gxx
def test_dobj_on_the_axes_is_the_sensitivity_at_the_vertex():
    import sensitivity_numpy as SN
    import harness_ranging as H
    for name in ("c2", "nuclear", "wind_battery_pem"):
        s, v = _bases(name)
        out = _ranging(s, v, None, None)
        dc, dr = H.axes(s.t)
        g = SN.sensitivities(s.t, s.cparams, s.rparams, v["x"], v["y"], v["status"])
        grad = np.concatenate([g[1] if s.t.Pc else np.zeros((len(s), 0)), g[2] if s.t.Pr else np.zeros((len(s), 0))], axis=1)
        scale = np.maximum(1.0, np.abs(grad).max(1, keepdims=True))
        assert (np.abs(out["dobj"] - grad) <= 1e-7 * scale).all(), (name, np.abs(out["dobj"] - grad).max())
        assert (out["d2obj"] == 0).all()                    # an axis moves c or b / u, never both


@needs_gxx
@pytest.mark.parametrize("case", ["free_wind", "solar_design_pv"])
def test_directions_that_move_A_are_nan(case):
    import harness_crossover as HX
    import harness_ranging as H
    if case == "free_wind":
        T, N = 24, 4
        lmp, cf, _, _ = SC.c2(N)
        t = TP.wind_battery_design_free_wind(T, None, 10000.0)
        cp = lmp
        rp = np.ascontiguousarray(np.broadcast_to(np.asarray(cf, float)[..., :T], (N, T)) - TP.CF_NOMINAL)
        status, x, y = interior_xy(type("Set", (), dict(t=t, cparams=cp, rparams=rp, __len__=lambda self: N))())
        v = HX.run(t, cp, rp, status, x, y)
    else:
        s, v = _bases(case)
        t, cp, rp = s.t, s.cparams, s.rparams
    assert (v["status"] == 0).all()
    out = H.run(t, cp, rp, v["status"], v["col_status"], v["row_basic"])
    in_A = np.zeros(t.Pr, bool)
    in_A[np.asarray(t.amap[2], int)] = True
    moves = np.concatenate([np.zeros(t.Pc, bool), in_A])
    assert moves.any() and not moves.all()
    for f in ("lo", "hi", "dobj", "d2obj"):
        assert np.isnan(out[f][:, moves]).all(), f
        assert not np.isnan(out[f][:, ~moves]).any(), f


@needs_gxx
def test_bad_bases_and_non_optimal_inputs():
    import harness_ranging as H
    s, v = _bases("c2")
    st = np.array([0, 1, 2, 3, 0, 0, 0, 0], np.int32)
    cs, rb = v["col_status"].copy(), v["row_basic"].copy()
    j = int(np.flatnonzero(cs[4] == 1)[0]); cs[4, j] = 0                      # m - 1 members
    j = int(np.flatnonzero(cs[5] == 0)[0]); cs[5, j] = 1                      # m + 1 members
    out = H.run(s.t, s.cparams, s.rparams, st, cs, rb)
    assert list(out["status"]) == [0, 1, 2, 3, 2, 2, 0, 0]
    bad = out["status"] != 0
    for f in ("lo", "hi", "dobj", "d2obj"):
        assert np.isnan(out[f][bad]).all() and not np.isnan(out[f][~bad]).any()
    assert (out["lo"][~bad] <= 0).all() and (out["hi"][~bad] >= 0).all()


@needs_gxx
def test_shared_and_per_lp_directions_agree_and_batch_position():
    import harness_ranging as H
    s, v = _bases("wind_battery_pem")
    dir_c, dir_r, _ = directions(s.t)
    a = H.run(s.t, s.cparams, s.rparams, v["status"], v["col_status"], v["row_basic"], dir_c, dir_r)
    N = len(s)
    b = H.run(s.t, s.cparams, s.rparams, v["status"], v["col_status"], v["row_basic"], np.broadcast_to(dir_c, (N,) + dir_c.shape),
              np.broadcast_to(dir_r, (N,) + dir_r.shape))
    k = np.array([3, 0, 3, 7, 1])
    c = H.run(s.t, s.cparams[k], s.rparams[k], v["status"][k], v["col_status"][k], v["row_basic"][k], dir_c, dir_r)
    for f in ("lo", "hi", "dobj", "d2obj", "status"):
        assert np.array_equal(a[f], b[f], equal_nan=True), f
        assert np.array_equal(a[f][k], c[f], equal_nan=True), f


@needs_gxx
def test_fixed_column_at_the_wrong_bound_blocks_where_the_direction_unfixes_it():
    """a column with u = 0 may sit at either bound; where a direction makes u positive and its reduced cost has the wrong sign for
    the bound it sits at, the basis stops being optimal at once on that side"""
    import harness_ranging as H
    T, N = 24, 4
    lmp, cf, W, _ = SC.c2(N, seed=5)
    t = TP.wind_battery_pem(T, with_battery=True)
    cp = np.ascontiguousarray(np.concatenate([lmp, np.full((N, 1), 2.5)], axis=1))
    rp = TP.wind_battery_rparams(T, cf, W, 0.0, pem_mw=200.0)           # no battery: its columns are fixed at 0 through Umap
    rp = np.ascontiguousarray(np.broadcast_to(rp, (N, t.Pr)))
    bases = []                                                            # HiGHS' bases (exact_lp.highs_basis)
    for k in range(N):
        c, b, u, _ = t.instantiate(cp[k], rp[k])
        A = t.matrix(rp[k]).tocsc(copy=True)
        A.sort_indices()
        bases.append(E.highs_basis(c, A, b, u))
    v = dict(col_status=np.array([q[0] for q in bases], np.int8), row_basic=np.array([q[1] for q in bases], np.int8),
             status=np.zeros(N, np.int32))
    gr = np.zeros((1, t.Pr)); gr[0, T] = 1e3                              # one more MW of battery
    gc = np.zeros((1, t.Pc))
    c, b, u, _ = t.instantiate(cp[0], rp[0])
    du = np.where(np.isfinite(u), t.Umap @ gr[0], 0.0)
    sd = np.abs(c).max()
    from oracle import ranging_numpy as RN
    flipped = 0
    for k in range(N):
        c, b, u, _ = t.instantiate(cp[k], rp[k])
        Bs = RN.Basis(t.matrix(rp[k]), b, c, u, v["col_status"][k], v["row_basic"][k])
        cand = np.flatnonzero((u <= 0) & (du != 0) & (v["col_status"][k] != 1) & (np.abs(Bs.d) > 1e-6 * sd))
        if not cand.size:
            continue
        cs = v["col_status"][[k]].copy()
        cs[0, cand[0]] = 2 - cs[0, cand[0]]                                  # the other bound: its d_j now has the wrong sign
        out = H.run(t, cp[[k]], rp[[k]], v["status"][[k]], cs, v["row_basic"][[k]], gc, gr)
        assert out["status"][0] == 0 and out["hi"][0, 0] == 0.0, (k, out["hi"])
        mr = RN.ranging(t, cp[k], rp[k], cs[0], v["row_basic"][k], gc, gr)
        assert mr["hi"][0] == 0.0
        basis = (cs[0], v["row_basic"][k].astype(bool))
        XR.verify(t, cp[k], rp[k], basis)                                     # optimal at theta = 0: the column is fixed
        assert XR.exact_range(t, cp[k], rp[k], basis, gc[0], gr[0])[1] == 0.0
        with pytest.raises(E.NotCertified):                                   # and not a little way along
            XR.verify(t, *XR.moved(t, cp[k], rp[k], gc[0], gr[0], 1e-3), basis)
        flipped += 1
    assert flipped >= 1
