"""The ranging kernel's outputs against a git revision's build (default HEAD~1), bit for bit, on the gpu_ranging_bench.py workloads (C4 cut
to 500 LPs): solve, crossover and ranging run once with each library, each in its own process with its own package.

    python tests/checks/ranging_parent_identity.py --prepare DIR [REV]    # needs git and nvcc, no GPU: DIR/<rev tree> with its library
    python tests/checks/ranging_parent_identity.py --compare DIR          # needs the GPU; prints one line, exits 1 on a difference
"""
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]

DUMP = r'''
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2] + "/tests"); sys.path.insert(0, sys.argv[2] + "/tests/checks")
from dispatches_b200 import solver as S
from gpu_crossover_bench import workloads
out = {}
for name, t, cp, rp, kw in workloads():
    cp = cp[:500] if name == "C4" else cp
    sol = S.BatchLPSolver(t, **kw)
    cpd = torch.as_tensor(np.ascontiguousarray(cp), device="cuda")
    if t.Pr and np.ndim(rp) == 2 and len(rp) == 1:
        rp = rp[0]
    if t.Pr and np.ndim(rp) == 2:
        rp = rp[:len(cp)]
    rpd = torch.as_tensor(np.ascontiguousarray(rp), device="cuda") if t.Pr else None
    r = sol.solve(cpd, rpd, want_x=True, want_y=True)
    v = sol.crossover(cpd, rpd, r)
    g = sol.ranging(cpd, rpd, v)
    for f in ("theta_lo", "theta_hi", "dobj", "d2obj", "status"):
        out[name + "_" + f] = getattr(g, f).cpu().numpy()
np.savez(sys.argv[3], **out)
'''


def prepare(d, rev):
    d = Path(d) / "parent"
    d.mkdir(parents=True, exist_ok=True)
    tar = subprocess.run(["git", "-C", str(ROOT), "archive", rev], check=True, capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", str(d)], input=tar, check=True)
    subprocess.run([sys.executable, "-m", "dispatches_b200.csrc.build"], cwd=d, check=True, capture_output=True)
    print("prepared", rev, "in", d)


def compare(d):
    import numpy as np
    with tempfile.TemporaryDirectory() as td:
        runs = {}
        for key, pkg in (("parent", Path(d) / "parent"), ("tree", ROOT)):
            f = Path(td) / f"{key}.npz"
            subprocess.run([sys.executable, "-c", DUMP, str(pkg), str(ROOT), str(f)], check=True)
            runs[key] = np.load(f)
        a, b = runs["parent"], runs["tree"]
        bad = [k for k in a.files if not np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8))]
    print(f"ranging outputs: {len(a.files)} arrays, {len(bad)} differ from the parent build" + (f": {bad}" if bad else ""))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    if sys.argv[1] == "--prepare":
        prepare(sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else "HEAD~1")
    else:
        compare(sys.argv[2])
