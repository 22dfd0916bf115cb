"""Every kernel family against the exact optima of real, degenerate dispatch LPs (tests/real_lps.py): stage 2, stage v1, the
long-horizon kernel, the storage-chain kernel and the band kernel, through check_exact -- objective, KKT residuals, x / y where
unique, and on every LP the columns every optimum has at a bound and the reduced costs every optimal y zeroes.

The launches are tiled as in test_stage_kernels_planted.py (2 x grid x problems_per_cta + 5 LPs in one launch, so that group
slots and warps take second and third tickets; every copy bitwise equal to its first), and the same launch-geometry asserts show which
kernel ran."""
import numpy as np
import pytest
import torch

import real_lps as R
from dispatches_b200 import solver as S
from planted_stage import CHAIN_T, chain_lanes, chain_smem_bytes
from test_kernel_status_parity import _assert_kernel
from dispatches_b200 import lp_template as LT

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def solve_device(sol, s, want_xy=True):
    """set s in ONE launch through the device call, results as numpy.  The host call cuts a pageable batch into chunks of about
    2 000 LPs, each its own launch, in which a group slot of a stage kernel rarely takes a second ticket."""
    dev = torch.device("cuda")
    r = sol.solve(torch.as_tensor(s.cparams, device=dev), torch.as_tensor(s.rparams, device=dev) if s.t.Pr else None,
                  want_x=want_xy, want_y=want_xy)
    torch.cuda.synchronize()
    return S.LPResult(*(None if a is None else a.cpu().numpy() for a in (r.obj, r.status, r.iters, r.x, r.y)))


def _run(s, sol, name, N=None, cperm=None, rperm=None, obj_rel=R.OBJ_REL):
    if N is None:
        big, _ = s.tile(40000)
        solve_device(sol, big, want_xy=False)
        N = 2 * S.last_launch()["grid"] * S.last_launch()["problems_per_cta"] + 5
    q, k = s.tile(N, seed=1)
    r = solve_device(sol, q)
    ll = S.last_launch()
    if name == "chain":
        # the chain kernel's own shared memory per warp and LPs per CTA (as in test_stage_kernels_planted._run)
        L, NF = chain_lanes(s.t.m), LT.detect_chain1(s.t)["NF"]
        warps = ll["block"] // 32
        assert sol.has_chain1 and ll["smem_bytes"] == chain_smem_bytes(NF) * warps, ll
        assert ll["problems_per_cta"] == (32 // L) * warps, ll
    elif name == "band":
        # one LP per warp, every SM busy (a stage-2 launch puts 32 / L LPs in a warp, a chain launch has its own shared memory)
        assert ll["problems_per_cta"] == ll["block"] // 32 and ll["grid"] == _sms(), ll
        assert not (sol.has_chain1 and ll["smem_bytes"] == chain_smem_bytes(LT.detect_chain1(s.t)["NF"]) * (ll["block"] // 32)), ll
    else:
        _assert_kernel(name, sol)
        if name == "stage_v1":
            assert ll["grid"] % _sms() == 0, ll
        elif name != "long":
            assert ll["grid"] == _sms(), ll
    first = np.unique(k, return_index=True)[1]
    for a in (r.obj, r.status, r.iters, r.x, r.y):
        assert np.array_equal(a, a[first[k]])
    e = R.check_exact(q, r.obj, r.status, r.x, r.y, cperm=cperm, rperm=rperm, kkt_rows=first, what=name, obj_rel=obj_rel)
    print(name, N, R.fmt(e))
    return q, r


STAGE2_T = [2, 5, 7, 12, 13, 23, 24, 31, 32, 33, 48, 49, 96]


@pytest.mark.parametrize("T", STAGE2_T)
def test_stage2_windows(T):
    s = R.windows(T)
    _run(s, S.BatchLPSolver(s.t), f"stage2_T{T}")


@pytest.mark.parametrize("name", ["c2", "c5", "edges"])
def test_stage2_batches(name):
    """C2 at a deterministic 1 024-LP stride, the strided C5 sample, and the edge set"""
    s = {"c2": lambda: R.c2(1024), "c5": R.c5, "edges": R.edges}[name]()
    _run(s, S.BatchLPSolver(s.t), "stage2_T24")


@pytest.mark.parametrize("T", [2, 13, 24, 32])
def test_stage_v1(T):
    s = R.windows(T)
    _run(s, S.BatchLPSolver(s.t, kernel=S.KERNEL_STAGE_V1), "stage_v1")


@pytest.mark.parametrize("T", [97, 128, 129, 168, 200])
def test_long(T):
    """no row may be bitwise the band kernel's result, or it would be testing the band kernel's retry pass"""
    s = R.windows(T)
    sol = S.BatchLPSolver(s.t)
    props = torch.cuda.get_device_properties(0)
    q, r = _run(s, sol, "long", N=2 * _sms() * (props.max_threads_per_multi_processor // 32) + 5)
    band = S.BatchLPSolver(s.t, kernel=S.KERNEL_BAND).solve_host(q.cparams, q.rparams, want_x=True, want_y=True)
    assert not (r.x == band.x).all(1).any() and not (r.y == band.y).all(1).any()


@pytest.mark.parametrize("report", [False, True], ids=["nuclear", "nuclear_report"])
@pytest.mark.parametrize("Lg", sorted(CHAIN_T))
def test_chain(Lg, report):
    """the descriptor set-up (the shuffled plain-CSR path is covered on planted chains in test_stage_kernels_planted.py)"""
    T = CHAIN_T[Lg]
    s = R.nuclear_report(T) if report else R.nuclear(T)
    sol = S.BatchLPSolver(s.t)
    assert sol.has_chain1
    _run(s, sol, "chain")


BAND = {"wb24": lambda: R.c2(64), "wb96": lambda: R.windows(96), "edges": R.edges, "pem": lambda: R.wind_battery_pem(24, True),
        "pem_nobatt": lambda: R.wind_battery_pem(24, False), "fossil": lambda: R.fossil(168), "design": R.design,
        **{o: (lambda o=o: R.operation(o)) for o in R.OPERATIONS}, **{f"solar_{z}": (lambda z=z: R.solar(z)) for z in R.SOLAR_SIZES}}


@pytest.mark.parametrize("name", sorted(BAND))
def test_band(name):
    s = BAND[name]()
    _run(s, S.BatchLPSolver(s.t, kernel=S.KERNEL_BAND), "band")
