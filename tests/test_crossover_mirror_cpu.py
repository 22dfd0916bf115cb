"""CPU tests of the numpy mirror of the crossover (oracle/crossover_numpy.py): from the numpy IPM mirrors' (x, y) its bases verify
as exact optima, and it is compared basis for basis with the kernel's source on the SIMT emulator.  The mirror follows the same rules
with different arithmetic (an LU solve of B from scratch for every step), so where a ratio test or pricing step meets a near tie the two
may pick different, equally valid vertices: the test reports every such LP and pins the sets where they agree everywhere."""
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

import exact_lp as E  # noqa: E402
import real_lps as R  # noqa: E402
from crossover_check import interior_xy  # noqa: E402
from oracle import crossover_numpy as XN  # noqa: E402

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ for the SIMT emulator")

# set: (make, dense IPM mirror, every LP's basis and pivot count equal to the emulated kernel's)
SETS = {
    "c2": (lambda: R.c2(16), False, True),
    "nuclear": (lambda: R.nuclear(24), False, True),
    "wind_battery_tracker": (lambda: R.operation("wind_battery_tracker"), False, False),
    "wind_battery_bidder_da": (lambda: R.operation("wind_battery_bidder_da"), False, False),
    "edges": (lambda: R.edges(), False, False),
    "design": (lambda: R.design(24), True, False),
}


def mirror(s, status, x):
    out = []
    for k in range(len(s)):
        if status[k] != 0:
            out.append(None)
            continue
        c, b, u, _ = s.t.instantiate(s.cparams[k], s.rparams[k])
        out.append(XN.crossover(s.t.matrix(s.rparams[k]), b, c, u, x[k]))
    return out


@needs_gxx
@pytest.mark.parametrize("name", sorted(SETS))
def test_mirror_vertices_are_exact_optima_and_match_the_kernel(name):
    import harness_crossover as H
    make, dense, all_equal = SETS[name]
    s = make()
    status, x, y = interior_xy(s, dense)
    v = H.run(s.t, s.cparams, s.rparams, status, x, y)
    differ = []
    for k, mr in enumerate(mirror(s, status, x)):
        if mr is None:
            continue
        assert mr["status"] == 0, (name, k)
        e = E.exact_optimum(s.t, s.cparams[k], s.rparams[k], basis=(mr["col_status"], mr["row_basic"].astype(bool)))
        assert abs(e.obj - s.obj[k]) <= 1e-9 * max(1.0, abs(s.obj[k]))
        if not (np.array_equal(mr["col_status"], v["col_status"][k]) and np.array_equal(mr["row_basic"], v["row_basic"][k])
                and mr["pivots"] == v["pivots"][k]):
            differ.append(k)
    print(name, "LPs where the mirror's vertex differs from the kernel's (both verified):", differ)
    if all_equal:
        assert differ == []
    assert len(differ) <= len(s) // 2, differ
