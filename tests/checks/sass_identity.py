"""Every kernel that exists at a git revision (default HEAD) compiles to the same SASS in the working tree: both sources are compiled
for sm_90a with the library's flags, and the SASS of every function is compared after the anonymous-namespace hash in mangled names
is normalised.  Functions only the working tree has (new kernels) are listed, not compared.  Needs nvcc, cuobjdump and git, no GPU.

    python tests/checks/sass_identity.py [REV]
"""
import re
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "tests" / "checks"))
from dense_sass_identity import CSRC, sass  # noqa: E402


def functions(text):
    out = {}
    for block in re.split(r"\n\s*Function : ", text)[1:]:
        name, body = block.split("\n", 1)
        key = re.sub(r"_(GLOBAL__N_|INTERNAL)_[0-9a-f]{8}_\d+_dsp_lp_cu_[0-9a-f]{8}", "ANON", name.strip())
        body = re.sub(r"_ZN\w+", "SYM", body)
        out[key] = [re.sub(r"/\*[0-9a-f]{4}\*/", "", l).strip() for l in body.splitlines() if l.strip()]
    return out


def main():
    rev = sys.argv[1] if len(sys.argv) > 1 else "HEAD"
    with tempfile.TemporaryDirectory() as td:
        td = Path(td)
        old = td / "old"; (old / CSRC).mkdir(parents=True); (old / "include").mkdir()
        files = subprocess.run(["git", "-C", str(ROOT), "ls-tree", "--name-only", rev, CSRC + "/"], check=True, capture_output=True,
                               text=True).stdout.split()
        for f in files + ["include/dsp_lp.h"]:
            (old / f).write_bytes(subprocess.run(["git", "-C", str(ROOT), "show", f"{rev}:{f}"], check=True, capture_output=True).stdout)
        (td / "a").mkdir(); (td / "b").mkdir()
        a = functions(sass(old / CSRC, old / "include", td / "a"))
        b = functions(sass(ROOT / CSRC, ROOT / "include", td / "b"))
    bad = [k for k in a if k not in b or a[k] != b[k]]
    new = [k for k in b if k not in a]
    print(f"{len(a)} functions at {rev}: {len(a) - len(bad)} identical, {len(bad)} different or missing; {len(new)} new")
    for k in new:
        print("  new:", k)
    for k in bad:
        print("  DIFFERENT:", k)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
