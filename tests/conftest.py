import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests need a CUDA device: on a CPU box they are skipped (a plain `pytest` run stays green)."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:            # noqa: BLE001
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device (the solver has no CPU fallback)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def cuda_solver_lib():
    """Builds (if needed) and loads the C-ABI library -- no compute."""
    from dispatches_b200.csrc import build
    build.build()
    from dispatches_b200 import solver
    return solver.load_library()
