"""The second attempt of the stage kernels' CUDA source on the lock-step SIMT emulator (tests/emu): stage 2 at every group width L,
the long-horizon kernel and the storage-chain kernel, on real LPs with certified exact optima (tests/real_lps.py).  The CPU half of
tests/test_second_attempt.py:

  * forced retry: with attempt 1 at step_frac FORCED no LP converges within max_iter, so every LP goes through attempt 2, which must
    end OPTIMAL in max_iter < iters <= 2 max_iter and pass check_exact;
  * restart independence: attempt 1 at FORCED_2 (also run to the cap) gives the same bits;
  * a mixed batch: at the first step_frac of test_second_attempt.LADDER where some LPs finish in attempt 1 and others need attempt 2,
    every LP is bitwise the same LP solved alone, so no group slot hands its next LP a stale attempt flag, iteration offset or reload
    mode.  The emulated warps run one after the other from one ticket counter, so each group slot of the first takes many LPs in turn."""
import importlib.util
import pathlib
import shutil

import numpy as np
import pytest

import real_lps as R
from dispatches_b200 import lp_template as LT

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")

MAX_ITER = 60
FORCED = 1e-3
FORCED_2 = 0.05
LADDER = tuple(round(0.30 + 0.01 * k, 2) for k in range(21))      # as in test_second_attempt.py
MIX_SHARE = 0.1
WARPS = 2


def _harness(name):
    spec = importlib.util.spec_from_file_location("emu_" + name, pathlib.Path(__file__).parent / "emu" / f"{name}.py")
    h = importlib.util.module_from_spec(spec); spec.loader.exec_module(h)
    h.build()
    return h


@pytest.fixture(scope="module")
def emu():
    return _harness("harness")


@pytest.fixture(scope="module")
def emc():
    return _harness("harness_chain1")


# group width L -> (T, P, N): a horizon the library runs on stage2::warp_body<L, P>, and the size of the mixed set (several LPs per
# group slot: a warp holds 32 / L groups)
STAGE2 = {2: (5, 3, 64), 4: (12, 3, 64), 8: (24, 3, 64), 16: (48, 3, 32), 32: (96, 3, 16)}


def _stage2(emu, L):
    T, P, _ = STAGE2[L]
    return lambda s, **kw: emu.solve(s.t, s.cparams, s.rparams, L, P, warps=WARPS, **kw)


def _long(emu):
    return lambda s, **kw: emu.solve_long(s.t, s.cparams, s.rparams, warps=WARPS, **kw)


def _chain(emc, L):
    return lambda s, **kw: emc.solve(s.t, LT.detect_chain1(s.t), s.cparams, s.rparams if s.t.Pr else None, L, 3, warps=WARPS, **kw)


def _forced(solve, s, what):
    obj, status, iters, x, y = out = solve(s, step_frac=FORCED)
    assert ((iters > MAX_ITER) & (iters <= 2 * MAX_ITER)).all(), (what, iters)
    e = R.check_exact(s, obj, status, x, y, what=what)
    again = solve(s, step_frac=FORCED_2)
    assert (again[2] > MAX_ITER).all(), (what, again[2])
    for a, b in zip(out, again):
        assert np.array_equal(a, b), what
    print(what, "iters", iters.min(), "..", iters.max(), R.fmt(e))


def _mixed(solve, s, what):
    seen = []
    for sf in LADDER:
        out = solve(s, step_frac=sf)
        a1, a2 = int((out[2] <= MAX_ITER).sum()), int((out[2] > MAX_ITER).sum())
        seen.append((sf, a1, a2))
        if min(a1, a2) >= MIX_SHARE * len(s):
            break
    else:
        pytest.fail(f"{what}: no step_frac of the ladder mixes first- and second-attempt LPs (>= {MIX_SHARE:.0%} each) on {len(s)} "
                    f"LPs: (step_frac, attempt 1, attempt 2) = {seen}")
    R.check_exact(s, out[0], out[1], out[3], out[4], what=what)
    for k in range(len(s)):
        solo = solve(s.take([k]), step_frac=sf)
        for a, b in zip(out, solo):
            assert np.array_equal(a[k], b[0]), (what, sf, k)
    print(what, f"step_frac {sf}: {a1} LPs finish in attempt 1, {a2} need attempt 2")


@pytest.mark.parametrize("L", sorted(STAGE2))
def test_stage2_forced_retry(emu, L):
    _forced(_stage2(emu, L), R.windows(STAGE2[L][0]), f"stage2 L{L}")


@pytest.mark.parametrize("L", sorted(STAGE2))
def test_stage2_mixed_batch(emu, L):
    T, _, N = STAGE2[L]
    _mixed(_stage2(emu, L), R.windows(T, N), f"stage2 L{L}")


def test_long_forced_retry(emu):
    _forced(_long(emu), R.windows(97, 4), "long")


def test_long_mixed_batch(emu):
    _mixed(_long(emu), R.windows(97, 8), "long")


@pytest.mark.parametrize("report", [False, True], ids=["nuclear", "nuclear_report"])
def test_chain_forced_retry(emc, report):
    s = R.nuclear_report(48, 8) if report else R.nuclear(48, 8)
    _forced(_chain(emc, 16), s, "chain")


def test_chain_mixed_batch(emc):
    _mixed(_chain(emc, 16), R.nuclear(48, 32), "chain")
