"""tools/stage2_critical_path.py on the built library: the SASS of the headline kernel splits into all nine phases of a round,
each with instructions and a dependent path (CPU only: cuobjdump / nvdisasm of the sm_90a code)."""
import importlib.util
import shutil
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _tool():
    spec = importlib.util.spec_from_file_location("stage2_critical_path", ROOT / "tools" / "stage2_critical_path.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.skipif(not (shutil.which("nvdisasm") or Path("/usr/local/cuda/bin/nvdisasm").exists()), reason="needs the CUDA toolkit")
def test_report_finds_all_phases(capsys):
    from dispatches_b200.csrc import build
    lib = build.build()
    cp = _tool()
    res = cp.main(["--lib", str(lib), "--chains", "3"])
    out = capsys.readouterr().out
    assert "MODEL" in out
    assert len(cp.PHASES) == 9
    for ph in cp.PHASES:
        assert res[ph]["insns"] > 0, ph
        assert res[ph]["path"] > 0, ph
    # the FP64 work of a round is in the passes, and every phase of the solve has shuffles
    assert sum(res[ph]["fp64"] for ph in cp.PHASES) > 3000
    for ph in ("factor + pred. solve", "pass 3 + corr. solve"):
        assert res[ph]["shfl"] > 0, ph
