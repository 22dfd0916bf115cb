"""obj / status / iters of all 560 640 C5 LPs (bench.config_data("C5")) from the library named by DSP_LP_LIB (default: the in-tree
build), as DIR/c5_{obj,status,iters}.npy: two builds compared output for output.  C2's counterpart is bench.py --dump-outputs.

    python tools/gpu_dump_c5.py DIR
    python tools/gpu_dump_c5.py --compare DIR_A DIR_B
"""
import os
import sys

sys.path.insert(0, ".")
import numpy as np


def compare(da, db):
    a = {k: np.load(os.path.join(da, f"c5_{k}.npy")) for k in ("obj", "status", "iters")}
    b = {k: np.load(os.path.join(db, f"c5_{k}.npy")) for k in ("obj", "status", "iters")}
    d_it = np.flatnonzero(a["iters"] != b["iters"])
    d_st = np.flatnonzero(a["status"] != b["status"])
    ok = np.isfinite(a["obj"]) & np.isfinite(b["obj"])
    rel = np.abs(a["obj"][ok] - b["obj"][ok]) / np.maximum(1.0, np.abs(a["obj"][ok]))
    print(f"C5 {a['obj'].size} LPs: iters differ {d_it.size}, status differ {d_st.size}, obj bitwise equal "
          f"{int((a['obj'] == b['obj']).sum())}, max rel obj diff {rel.max() if rel.size else 0.0:.2e}")
    for i in d_it[:20]:
        print(f"   LP {i}: iters {a['iters'][i]} -> {b['iters'][i]}, status {a['status'][i]} -> {b['status'][i]}")


def dump(out):
    import torch
    from bench import config_data
    from dispatches_b200 import solver as S
    build_t, cp, rp, _ = config_data("C5")
    dev = torch.device("cuda", 0)
    sol = S.BatchLPSolver(build_t())
    r = sol.solve(torch.tensor(cp, device=dev), torch.tensor(rp, device=dev))
    torch.cuda.synchronize()
    os.makedirs(out, exist_ok=True)
    for k in ("obj", "status", "iters"):
        np.save(os.path.join(out, f"c5_{k}.npy"), getattr(r, k).cpu().numpy().astype(np.float64))
    print(f"C5 {cp.shape[0]} LPs -> {out}: iters mean {float(r.iters.float().mean()):.3f}, non-optimal {int((r.status != 0).sum())},"
          f" launch {S.last_launch()}")


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        compare(sys.argv[2], sys.argv[3])
    else:
        dump(sys.argv[1])
