"""The dense kernel (dsp_ipm_dense_kernel, csrc/dsp_dense.cuh) against the exact optima of real, degenerate LPs (tests/real_lps.py)
through check_exact -- objective, KKT residuals, x / y where unique, and on every LP the columns every optimum has at a bound and
the reduced costs every optimal y zeroes -- with the planted suite's bars:

  * its own templates: the PV + battery + hydrogen design LP, baked (one PV series) and with a PV series per LP (the PerLP
    instantiation), at T = 24 and 48;
  * DSP_KERNEL_DENSE on band templates: every set of test_real_lps_exact.BAND (the fixed-size PV + battery + hydrogen LPs among
    them), C2, C5, nuclear and nuclear_report at T = 48, and wind + battery windows whose m = 4T sits on the 64-row tile edges, up
    to m = 1024.

Each launch holds 2 x grid + 5 LPs (the grid of a launch with more LPs than fit), every copy bitwise equal to its first, and the
launch geometry (256 threads, one LP per CTA) shows that the dense kernel ran."""
import numpy as np
import pytest
import torch

import real_lps as R
from dispatches_b200 import solver as S
from test_real_lps_exact import BAND

pytestmark = pytest.mark.gpu

THREADS = 256                        # kDenseWarps x 32


def _grid(s):
    """the grid of a dense launch with more LPs than fit (8 per SM: at most 8 CTAs of 256 threads are resident on an SM); the
    geometry does not depend on max_iter, so that launch runs one iteration"""
    big, _ = s.tile(8 * torch.cuda.get_device_properties(0).multi_processor_count)
    S.BatchLPSolver(s.t, kernel=S.KERNEL_DENSE, max_iter=1).solve_host(big.cparams, big.rparams if s.t.Pr else None)
    return S.last_launch()["grid"]


def _run(s, name):
    N = 2 * _grid(s) + 5
    q, k = s.tile(N, seed=1)
    r = S.BatchLPSolver(s.t, kernel=S.KERNEL_DENSE).solve_host(q.cparams, q.rparams if s.t.Pr else None, want_x=True, want_y=True)
    ll = S.last_launch()
    assert ll["block"] == THREADS and ll["problems_per_cta"] == 1 and ll["grid"] == (N - 5) // 2, ll
    first = np.unique(k, return_index=True)[1]
    for a in (r.obj, r.status, r.iters, r.x, r.y):
        assert np.array_equal(a, a[first[k]])
    e = R.check_exact(q, r.obj, r.status, r.x, r.y, kkt_rows=first, what=name)
    print(name, N, f"iters mean {r.iters.mean():.1f} max {r.iters.max()}", R.fmt(e))
    return e


NATIVE = {"solar_design24": lambda: R.solar_design(24), "solar_design48": lambda: R.solar_design(48),
          "solar_design_pv24": lambda: R.solar_design_pv(24), "solar_design_pv48": lambda: R.solar_design_pv(48)}


@pytest.mark.parametrize("name", sorted(NATIVE))
def test_dense_templates(name):
    s = NATIVE[name]()
    assert s.t.w > 32 and (s.t.amap is not None) == ("_pv" in name)
    _run(s, name)


TILE_EDGE_T = [16, 17, 32, 33, 256]          # wind_battery(T): m = 4T = 64, 68, 128, 132 and 1024 (the dense kernel's limit)

ON_BAND = {**BAND, "c2": lambda: R.c2(1024), "c5": R.c5, "nuclear48": lambda: R.nuclear(48),
           "nuclear_report48": lambda: R.nuclear_report(48), **{f"wb{T}": (lambda T=T: R.windows(T)) for T in TILE_EDGE_T}}


@pytest.mark.parametrize("name", sorted(ON_BAND))
def test_dense_kernel_on_band_templates(name):
    s = ON_BAND[name]()
    assert s.t.w <= 32
    if name.startswith("wb") and name[2:].isdigit():
        assert s.t.m == 4 * int(name[2:])
    _run(s, name)
