"""The stage kernels that carry the workload -- stage 2 (several LPs per warp), stage v1 (lane per period), the long-horizon kernel
and the storage-chain kernel -- against exact optima (tests/planted_stage.py, tests/exact_lp.py): objective, x and y element by
element in the caller's order, and the KKT residuals of every LP, at every geometry each family is instantiated for.

Each case tiles a pool of certified LPs, in a random permutation, to 2 x grid x problems_per_cta + 5 LPs of a full launch: more
than two waves of full CTAs, every LP group refilled and every slot reused.  Every copy of an LP must equal its first copy
bitwise, so the KKT residuals are measured on the first copies only."""
import functools

import numpy as np
import pytest
import torch

from dispatches_b200 import lp_template as LT
from dispatches_b200 import solver as S
from planted_lp import shuffled
from planted_stage import CHAIN_T, CHAIN_VARIANTS, chain_lanes, chain_smem_bytes, check, planted_chain, planted_wb
from test_kernel_status_parity import _assert_kernel

pytestmark = pytest.mark.gpu

POOL = 64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(p, sol, name, N=None, t=None, cperm=None, rperm=None):
    """solves the pool tiled to N LPs -- by default 2 x grid x problems_per_cta + 5 of a launch that fills every SM (a probe batch
    of 40 000 LPs gives that geometry) -- and checks every LP against its exact optimum"""
    if N is None:
        big, _ = p.tile(40000)
        sol.solve_host(big.cparams, big.rparams)
        N = 2 * S.last_launch()["grid"] * S.last_launch()["problems_per_cta"] + 5
    q, k = p.tile(N, seed=1)
    r = sol.solve_host(q.cparams, q.rparams, want_x=True, want_y=True)
    ll = S.last_launch()
    if name == "chain":
        # the chain kernel's own shared memory per warp, which no band-kernel placement matches (at L = 32 its problems_per_cta is
        # one per warp, like the band kernel's, so the status tests' helper cannot tell the two apart there)
        L, NF = chain_lanes(p.t.m), LT.detect_chain1(p.t)["NF"]
        warps = ll["block"] // 32
        assert sol.has_chain1 and ll["smem_bytes"] == chain_smem_bytes(NF) * warps, ll
        assert ll["problems_per_cta"] == (32 // L) * warps, ll
    else:
        _assert_kernel(name, sol)
    if name == "stage_v1":                # several CTAs per SM
        assert ll["grid"] % _sms() == 0, ll
    elif name != "long":                  # (the long kernel's last launch is the band kernel's retry pass)
        assert ll["grid"] == _sms(), ll
    first = np.unique(k, return_index=True)[1]          # first[v]: index of the first copy of pool LP v
    for a in (r.obj, r.status, r.iters, r.x, r.y):
        assert np.array_equal(a, a[first[k]])
    err = check(q, r.obj, r.status, r.x, r.y, t=t, cperm=cperm, rperm=rperm, kkt_rows=first, what=name)
    print(name, N, {a: f"{b:.1e}" for a, b in err.items()})
    return q, r


@functools.lru_cache(maxsize=None)
def _wb(T):
    p = planted_wb(T, POOL, seed=11)
    assert p.x_margin > 1e-2 and p.r_margin > 1e-3, (p.x_margin, p.r_margin)      # what XY_REL assumes (planted_stage.py)
    return p


@pytest.mark.parametrize("T", [2, 5, 7, 12, 13, 23, 24, 31, 32, 33, 48, 49, 96])
def test_stage2(T):
    p = _wb(T)
    sol = S.BatchLPSolver(p.t)
    _run(p, sol, f"stage2_T{T}")


@pytest.mark.parametrize("T", [13, 24, 96])
def test_stage2_full_battery(T):
    p = planted_wb(T, POOL, seed=12, soc=True)
    _run(p, S.BatchLPSolver(p.t), f"stage2_T{T}")


@pytest.mark.parametrize("T", [2, 13, 24, 32])
def test_stage_v1(T):
    p = _wb(T)
    _run(p, S.BatchLPSolver(p.t, kernel=S.KERNEL_STAGE_V1), "stage_v1")


@pytest.mark.parametrize("T", [97, 128, 129, 200])
def test_long(T):
    """the long kernel (one warp per LP) runs with the band kernel's retry pass behind it, which re-solves every LP the long kernel
    left non-optimal: no row may be bitwise the KERNEL_BAND result, or that row would be testing the retry pass.

    The last launch is the retry pass, so the long kernel's geometry cannot be read back; the batch is sized from the device's
    limit instead: the long kernel keeps at most sm_count x occupancy x 4 warps resident, one LP each, and no occupancy can
    exceed max_threads_per_multi_processor / 32 warps per SM, so 2 x SMs x that + 5 LPs is more than two waves."""
    p = _wb(T)
    sol = S.BatchLPSolver(p.t)
    props = torch.cuda.get_device_properties(0)
    q, r = _run(p, sol, "long", N=2 * _sms() * (props.max_threads_per_multi_processor // 32) + 5)
    band = S.BatchLPSolver(p.t, kernel=S.KERNEL_BAND).solve_host(q.cparams, q.rparams, want_x=True, want_y=True)
    assert not (r.x == band.x).all(1).any() and not (r.y == band.y).all(1).any()


def _chain_solver(p, native):
    if native:
        t, cperm, rperm = shuffled(p.t, seed=13)
        return S.BatchLPSolver(t, native_setup=True), t, cperm, rperm
    return S.BatchLPSolver(p.t), None, None, None


@pytest.mark.parametrize("native", [False, True], ids=["desc", "csr_shuffled"])
@pytest.mark.parametrize("bounded", ["mixed", "all", "none"])
@pytest.mark.parametrize("NF", [2, 3])
@pytest.mark.parametrize("Lg", sorted(CHAIN_T))
def test_chain(Lg, NF, bounded, native):
    """descriptor set-up, and a plain CSR template in a shuffled caller order (the kernel writes x / y back through x_perm /
    y_perm)"""
    p = planted_chain(CHAIN_T[Lg], NF, seed=14, N=POOL, bounded=bounded)
    sol, t, cperm, rperm = _chain_solver(p, native)
    assert sol.has_chain1
    _run(p, sol, "chain", t=t, cperm=cperm, rperm=rperm)


@pytest.mark.parametrize("native", [False, True], ids=["desc", "csr_shuffled"])
@pytest.mark.parametrize("name", sorted(CHAIN_VARIANTS))
def test_chain_scaled(name, native):
    p = planted_chain(24, 3, seed=15, N=POOL, **CHAIN_VARIANTS[name])
    sol, t, cperm, rperm = _chain_solver(p, native)
    assert sol.has_chain1
    _run(p, sol, "chain", t=t, cperm=cperm, rperm=rperm)
