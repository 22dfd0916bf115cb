"""Turns the ncu captures and launch CSVs the tools/ scripts wrote into small summaries under profiles/ (git-ignored; needs no GPU)."""
import csv, collections, json, subprocess, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "profiles"; OUT.mkdir(exist_ok=True)
G = ROOT / "gpurun_out"

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
        "launch__waves_per_multiprocessor", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores",
        "smsp__pcsamp_warps_issue_stalled_wait", "smsp__pcsamp_warps_issue_stalled_short_scoreboard",
        "smsp__pcsamp_warps_issue_stalled_long_scoreboard", "smsp__pcsamp_warps_issue_stalled_math_pipe_throttle",
        "smsp__pcsamp_warps_issue_stalled_not_selected", "smsp__pcsamp_warps_issue_stalled_selected",
        "smsp__pcsamp_warps_issue_stalled_branch_resolving", "smsp__pcsamp_warps_issue_stalled_no_instructions",
        "smsp__pcsamp_warps_issue_stalled_barrier", "smsp__pcsamp_warps_issue_stalled_mio_throttle"]


def raw(rep):
    txt = subprocess.run(["ncu", "-i", str(rep), "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    return dict(zip(rows[0], zip(rows[1], rows[2])))


def opcode_mix(rep, n_lp):
    txt = subprocess.run(["ncu", "-i", str(rep), "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    hdr = rows[1]; ia = hdr.index("Instructions Executed"); isrc = hdr.index("Source")
    cnt = collections.Counter()
    for r in rows[2:]:
        if len(r) <= ia: continue
        op = r[isrc].strip().split()
        if not op: continue
        o = op[1] if op[0].startswith("@") else op[0]
        cnt[o.split(".")[0]] += int(r[ia])
    tot = sum(cnt.values())
    return {"warp_instructions_per_lp": tot / n_lp, "mix_pct": {k: round(100 * v / tot, 1) for k, v in cnt.most_common(14)}}


def summarize(name, rep, n_lp=10000):
    d = raw(rep)
    out = {"report": rep.name, "kernel": name, "lps_in_launch": n_lp}
    for k in KEYS:
        if k in d:
            out[k] = {"unit": d[k][0], "value": d[k][1]}
    out["traffic_bytes_per_launch"] = float(d["dram__bytes_read.sum"][1]) * {"Mbyte": 1e6, "Kbyte": 1e3, "byte": 1, "Gbyte": 1e9}[d["dram__bytes_read.sum"][0]] + \
        float(d["dram__bytes_write.sum"][1]) * {"Mbyte": 1e6, "Kbyte": 1e3, "byte": 1, "Gbyte": 1e9}[d["dram__bytes_write.sum"][0]]
    out.update(opcode_mix(rep, n_lp))
    json.dump(out, open(OUT / f"{rep.stem}.summary.json", "w"), indent=1)
    print(rep.name, out["gpu__time_duration.sum"], "issue%", out["smsp__issue_active.avg.pct_of_peak_sustained_active"]["value"],
          "fp64%", out["sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active"]["value"], "instr/LP", round(out["warp_instructions_per_lp"]))


def launches(csvfile, dst):
    rows = [r for r in csv.reader(open(csvfile)) if len(r) > 10 and r[0].isdigit()]
    agg = collections.defaultdict(list)
    for r in rows:
        agg[r[4].split("(")[0][-60:]].append(float(r[-1]) * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "usecond": 1.0, "nsecond": 1e-3, "msecond": 1e3}.get(r[-2], 1.0))
    tot = sum(sum(v) for v in agg.values())
    with open(dst, "w") as f:
        f.write("kernel,launches,total_us,mean_us,share_pct\n")
        for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
            f.write(f"{k},{len(v)},{sum(v):.1f},{sum(v)/len(v):.1f},{100*sum(v)/tot:.1f}\n")
    print(open(dst).read())


if __name__ == "__main__":
    for name, rep, nlp in (("dsp_ipm_band_kernel<4> (C2, first version)", G / "prof_r1_band.ncu-rep", 10000),
                           ("dsp_ipm_stage_wb_kernel (C2, first 168-register version)", G / "prof_r1_stage_v2.ncu-rep", 10000),
                           ("dsp_ipm_stage_wb_kernel (C2, final round-1 version)", G / "prof_r1_stage_final.ncu-rep", 10000),
                           ("dsp_ipm_band_kernel<1> (C3 nuclear template, 32 LPs, final round-1 version)", G / "prof_r1_band_final.ncu-rep", 32)):
        if rep.exists():
            summarize(name, rep, nlp)
    if (G / "launches_r1.csv").exists():
        launches(G / "launches_r1.csv", OUT / "launches_r1.csv")
