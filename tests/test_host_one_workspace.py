"""A host call whose kernel runs in the handle's one global workspace takes the batch in one chunk: chunk kernels on the handle's two
streams would index the same per-warp regions of that workspace at once.  The split band kernel on a pageable batch large enough to be
cut into chunks must give what the device call on the same batch gives, bit for bit.  The template's band kernel runs with its work
regions in shared memory, so the band kernel's placement alone does not keep the batch in one piece."""
import numpy as np
import pytest

from dispatches_b200 import solver as S
from planted_lp import band_placement, planted

pytestmark = pytest.mark.gpu


def test_split_kernel_host_call_of_4096_pageable_lps_runs_in_one_chunk():
    import torch
    p = planted(m=128, w=2, extra=0, bounded="none", seed=11, N=4096)
    assert band_placement(p.t)[0] == "smem_staged"
    sol = S.BatchLPSolver(p.t, kernel=S.KERNEL_BAND_SPLIT)
    ref = sol.solve(torch.from_numpy(p.cparams).cuda(), torch.from_numpy(p.rparams).cuda(), want_x=True)
    torch.cuda.synchronize()
    n0 = S.launch_count()
    r = sol.solve_host(p.cparams, p.rparams, want_x=True)
    assert S.launch_count() - n0 == 2          # one chunk: the split kernel, then the band kernel's retry pass
    for f in ("obj", "status", "iters", "x"):
        assert np.array_equal(getattr(r, f), getattr(ref, f).cpu().numpy()), f
