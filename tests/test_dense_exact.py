"""The dense kernels against the exact optima of real, degenerate LPs (tests/real_lps.py) through check_exact -- objective, KKT
residuals, x / y where unique, and on every LP the columns every optimum has at a bound and the reduced costs every optimal y zeroes
-- with the planted suite's bars.  The single-CTA kernel (dsp_ipm_dense_kernel, m <= 1024) and the cluster kernel
(dsp_ipm_dense_cluster_kernel, m <= 4096, one LP per cluster of 4 or 8 CTAs) run:

  * their own templates: the PV + battery + hydrogen design LP, baked (one PV series) and with a PV series per LP (the PerLP
    instantiation), at T = 24 and 48 on both kernels, and at T = 72, 96 (clusters of 4) and 168 (clusters of 8) on the cluster kernel;
  * DSP_KERNEL_DENSE / _DENSE_CLUSTER on band templates: every set of test_real_lps_exact.BAND (the fixed-size PV + battery + hydrogen
    LPs among them), C2, C5, nuclear and nuclear_report at T = 48, and wind + battery windows whose m = 4T sits on the 64-row tile
    edges up to m = 1024; on the cluster kernel also m = 1028 (past the single-CTA limit), 2048 (the last size on clusters of 4), 2052
    (the first on clusters of 8) and 4096 (its limit);
  * LPs whose rows and columns come in an order other than the template's (planted_lp.shuffled): the permutation that writes x
    back in the caller's order, and the per-problem matrix terms placed by CSR position in the caller's order.

Each launch holds 2 x (CTAs or clusters in flight) + 5 LPs, so CTAs and clusters take second and third tickets; every copy must be
bitwise equal to its first (a cluster that reads a tile another rank has not finished, keeps state from its previous ticket or loads a
per-problem value over another LP's perturbs the rounding long before the answer).  The launch geometry shows which kernel ran, and on
the cluster kernel its shared memory shows where the per-LP vectors sit.  Where both kernels run (m <= 1024) the cluster kernel's
status, objective, iterations, x and y are bitwise the single-CTA kernel's: it runs the same iteration, and its cluster factorisation
and substitutions are bitwise the single-CTA routines (test_dense_cluster_cpu.py)."""
import numpy as np
import pytest
import torch

import real_lps as R
from dispatches_b200 import solver as S
from dispatches_b200 import templates as TP
from oracle.highs import host_cores
from planted_lp import planted, shuffled
from test_real_lps_exact import BAND

pytestmark = pytest.mark.gpu

THREADS = 256                        # kDenseWarps x 32
KERNELS = {"dense": S.KERNEL_DENSE, "cluster": S.KERNEL_DENSE_CLUSTER}
MAX_M = {"dense": 1024, "cluster": 4096}
TS = 64                              # tile edge
# kDenseClusterSmemFixed: the reduction slots of 8 warps, one staged tile and kGroup = 2 target and operand tiles (row stride 65)
CLUSTER_SMEM_FIXED = (2 * 8 + 5 * TS * (TS + 1)) * 8


def _cluster_size(m):
    return 4 if -(-m // TS) <= 32 else 8


def _cluster_smem(t):
    """(dynamic shared memory of a cluster launch, whether the per-LP vectors sit in it): they do when they fit next to the tile
    buffers, else each rank keeps them in its workspace region (launch_dense_cluster)"""
    nt = -(-t.m // TS)
    vec = 8 * (8 * t.n + 6 * int(np.isfinite(t.u0).sum()) + 3 * t.m + 2 * nt * TS)
    fits = CLUSTER_SMEM_FIXED + vec <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    return CLUSTER_SMEM_FIXED + (vec if fits else 0), fits


def _units(t, s, kernel):
    """CTAs (dense) or clusters (cluster) in flight in a launch of s on template t with more LPs than fit (8 per SM); the geometry
    does not depend on max_iter, so that launch runs one iteration"""
    big, _ = s.tile(8 * torch.cuda.get_device_properties(0).multi_processor_count)
    S.BatchLPSolver(t, kernel=KERNELS[kernel], max_iter=1).solve_host(big.cparams, big.rparams if t.Pr else None)
    ll = S.last_launch()
    return ll["grid"] // ll["problems_per_cta"]


def _run(s, name, kernel, t=None, cperm=None, rperm=None, opts={}):
    """s through one dense kernel with solver options ``opts``, on s.t or on ``t``, the same LPs with column j / row i being column
    cperm[j] / row rperm[i] of s.t; on the cluster kernel at m <= 1024 also through the single-CTA kernel, which must give the same
    bits.  Returns the tiled set and the result."""
    t = s.t if t is None else t
    units = _units(t, s, kernel)
    N = 2 * units + 5
    q, k = s.tile(N, seed=1)
    rp = q.rparams if t.Pr else None
    r = S.BatchLPSolver(t, kernel=KERNELS[kernel], **opts).solve_host(q.cparams, rp, want_x=True, want_y=True)
    ll = S.last_launch()
    ppc = 1 if kernel == "dense" else _cluster_size(t.m)
    assert ll["block"] == THREADS and ll["problems_per_cta"] == ppc and ll["grid"] == ppc * units and units < N, ll
    placement = ""
    if kernel == "cluster":
        smem, fits = _cluster_smem(t)
        assert ll["smem_bytes"] == smem, (ll, smem)
        placement = f", clusters of {ppc}, vectors in {'shared memory' if fits else 'the workspace'}"
    first = np.unique(k, return_index=True)[1]
    for a in (r.obj, r.status, r.iters, r.x, r.y):
        assert np.array_equal(a, a[first[k]])
    e = R.check_exact(q, r.obj, r.status, r.x, r.y, cperm=cperm, rperm=rperm, kkt_rows=first, what=name)
    same = ""
    if kernel == "cluster" and t.m <= MAX_M["dense"]:
        d = S.BatchLPSolver(t, kernel=S.KERNEL_DENSE, **opts).solve_host(q.cparams, rp, want_x=True, want_y=True)
        for what in ("status", "obj", "iters", "x", "y"):
            assert np.array_equal(getattr(r, what), getattr(d, what)), (name, what, "differs from the single-CTA kernel")
        same = ", bitwise the single-CTA kernel's"
    print(f"{name} on the {kernel} kernel: m = {t.m}, {N} LPs{placement}, iters mean {r.iters.mean():.1f} max {r.iters.max()}{same}",
          R.fmt(e))
    return q, r


def _design(T, pv, N):
    """the design sets; the long horizons take tens of seconds per LP to certify, so they certify on every core"""
    procs = 1 if T <= 48 else host_cores()
    return R.solar_design_pv(T, N, procs=procs) if pv else R.solar_design(T, N, procs=procs)


# T: (N baked, N with a PV series per LP); the PV sets need N >= 6 for their six cases.  m = 15 T + 3.
DESIGN_T = {24: (8, 8), 48: (8, 8), 72: (8, 8), 96: (8, 6), 168: (2, 6)}
NATIVE = {f"solar_design{'_pv' if pv else ''}{T}": (T, pv) for T in DESIGN_T for pv in (False, True)}


def _native(name, kernel):
    T, pv = NATIVE[name]
    s = _design(T, pv, DESIGN_T[T][pv])
    assert s.t.m == 15 * T + 3 and s.t.w > 32 and (s.t.amap is not None) == pv
    _run(s, name, kernel)


@pytest.mark.parametrize("name", sorted(n for n, (T, _) in NATIVE.items() if 15 * T + 3 <= MAX_M["dense"]))
def test_dense_templates(name):
    _native(name, "dense")


@pytest.mark.parametrize("name", sorted(NATIVE))
def test_cluster_templates(name):
    """T = 72 and 96 on clusters of 4, T = 168 on clusters of 8; on the PV sets consecutive tickets of a cluster carry different PV
    series, so dense_load_matrix must replace every value of the previous LP"""
    _native(name, "cluster")


TILE_EDGE_T = [16, 17, 32, 33, 256]          # wind_battery(T): m = 4T = 64, 68, 128, 132 and 1024 (the dense kernel's limit)
CLUSTER_EDGE_T = [257, 512, 513, 1024]       # m = 1028, 2048 (32 tile rows: clusters of 4), 2052 (clusters of 8), 4096 (the limit)

ON_BAND = {**BAND, "c2": lambda: R.c2(1024), "c5": R.c5, "nuclear48": lambda: R.nuclear(48),
           "nuclear_report48": lambda: R.nuclear_report(48), **{f"wb{T}": (lambda T=T: R.windows(T)) for T in TILE_EDGE_T}}
CLUSTER_ON_BAND = {**ON_BAND, **{f"wb{T}": (lambda T=T: R.windows(T)) for T in CLUSTER_EDGE_T}}


def _on_band(name, kernel):
    s = CLUSTER_ON_BAND[name]()
    assert s.t.w <= 32
    if name.startswith("wb") and name[2:].isdigit():
        assert s.t.m == 4 * int(name[2:])
    _run(s, name, kernel)


@pytest.mark.parametrize("name", sorted(ON_BAND))
def test_dense_kernel_on_band_templates(name):
    _on_band(name, "dense")


@pytest.mark.parametrize("name", sorted(CLUSTER_ON_BAND))
def test_cluster_kernel_on_band_templates(name):
    _on_band(name, "cluster")


def test_cluster_runs_both_vector_placements():
    """the sets above run both of the cluster kernel's vector placements: C2 (wind_battery(24), m = 96) with its vectors in shared
    memory, the 1024-hour windows (m = 4096) with them in the workspace"""
    assert _cluster_smem(TP.wind_battery(24))[1] and not _cluster_smem(TP.wind_battery(1024))[1]


SHUFFLED = {"planted1100": ("cluster",), "solar_design_pv24": ("dense", "cluster")}


@pytest.mark.parametrize("name,kernel", [(n, k) for n, ks in SHUFFLED.items() for k in ks])
def test_caller_order(name, kernel):
    """rows and columns in a random caller order (the dense set-up puts the bounded columns first, keeps the rows, and the kernels
    write x back in the caller's order): a planted LP past the single-CTA limit with w > 32, and the design LPs with a PV series per
    LP, whose per-problem matrix terms the set-up places by CSR position in the caller's order"""
    if name == "planted1100":
        p = planted(1100, 40, seed=8, N=4)
        s = R.certify(p.t, p.cparams, p.rparams, procs=host_cores())
    else:
        s = R.solar_design_pv(24)
    ts, cperm, rperm = shuffled(s.t, seed=5)
    assert ts.w > 32 and (ts.amap is not None) == (name != "planted1100")
    _run(s, name + "_shuffled", kernel, t=ts, cperm=cperm, rperm=rperm)
