"""The dense kernel's baked-matrix instantiation compiles to the same SASS as at a git revision (default HEAD): both sources are compiled
for sm_90a with the library's flags, and the SASS of the dense kernel is compared after the mangled names are normalised.  Needs nvcc,
cuobjdump and git, no GPU.

    python tests/checks/dense_sass_identity.py [REV]
"""
import re
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from dispatches_b200.csrc import build as B  # noqa: E402

CSRC = "dispatches_b200/csrc"


def sass(src_dir, inc_dir, out):
    cubin = out / "k.cubin"
    flags = [f for f in B.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC") and not f.startswith("-I")]
    subprocess.run([B.nvcc_path(), *flags, "-cubin", f"-I{inc_dir}", str(src_dir / "dsp_lp.cu"), "-o", str(cubin)], check=True,
                   capture_output=True)
    cuobjdump = str(Path(B.nvcc_path()).parent / "cuobjdump")
    return subprocess.run([cuobjdump, "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout


def dense_functions(text):
    """SASS of every dense-kernel function, keyed by a name with the anonymous-namespace hash and the template argument normalised"""
    out = {}
    for block in re.split(r"\n\s*Function : ", text)[1:]:
        name, body = block.split("\n", 1)
        if "dsp_ipm_dense_kernel" not in name:
            continue
        key = "dense<true>" if "ILb1E" in name else "dense<false>"
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
        a = dense_functions(sass(old / CSRC, old / "include", td / "a"))
        b = dense_functions(sass(ROOT / CSRC, ROOT / "include", td / "b"))
    base = a.get("dense<false>")
    new = b.get("dense<false>")
    assert base and new, (list(a), list(b))
    same = base == new
    print(f"dense kernel at {rev}: {len(base)} SASS lines; baked-matrix instantiation now: {len(new)} lines, "
          f"{'identical' if same else 'DIFFERENT'}; per-LP instantiation: {len(b.get('dense<true>', []))} lines")
    if not same:
        for i, (x, y) in enumerate(zip(base, new)):
            if x != y:
                print(f"first difference at line {i}:\n  {x}\n  {y}")
                break
        sys.exit(1)


if __name__ == "__main__":
    main()
