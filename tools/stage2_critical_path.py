"""Critical-path model of one round of the generation-2 stage kernel, phase by phase (runs on CPU, no GPU needed).

    python tools/stage2_critical_path.py                       # the built library (dispatches_b200/csrc/libdsp_lp.so)
    python tools/stage2_critical_path.py --compile [-D...]     # compile dsp_lp.cu for sm_90a into a temporary directory
    python tools/stage2_critical_path.py --cubin FILE.cubin    # any cubin built with -lineinfo
    ... [--kernel 8,3] [--chains 10] [--json OUT]

It disassembles `dsp_ipm_stage2_wb_kernel<L, P>` with its line information (`nvdisasm -gi`), assigns every SASS instruction to
the phase of the round whose source lines it was compiled from (the `// ====` markers of `warp_body` in dsp_stage2.cuh, and the
exit vote), builds the register dependency graph of each phase (read-after-write through general and predicate registers,
64-bit values as register pairs, load -> use through LDS / LDG / LDL / SHFL) and reports its longest weighted path.

THIS IS A MODEL, NOT A MEASUREMENT.  Each instruction costs the fixed latency of LATENCY below; a branch, convergence or barrier
instruction is a barrier (nothing after it starts before everything before it in its phase has finished); issue slots,
dual-issue limits, other warps, bank conflicts and memory ordering through shared memory are ignored.  Its job is to rank
where a round's dependent latency sits, and to show the change in chain length between two builds.  Cycles per phase on the
GPU come from tools/gpu_stage2_phases.py.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import subprocess
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "dispatches_b200" / "csrc"
STAGE2 = CSRC / "dsp_stage2.cuh"

# model latencies in cycles (dependent issue to dependent issue), by opcode without modifiers
LATENCY = {
    "DFMA": 8, "DADD": 8, "DMUL": 8, "DSETP": 8,          # FP64 pipe
    "MUFU": 20,                                          # MUFU.RCP64H, the reciprocal seed
    "SHFL": 30,
    "LDS": 30,
    "LDL": 30,                                           # spill reload (L1)
    "LDG": 300,                                          # global load (L2 hit or HBM)
    "LDC": 15, "ULDC": 15,
    "F2F": 8, "I2F": 8, "F2I": 8,
}
DEFAULT_LATENCY = 4                                      # integer / FP32 / select / move
BARRIER_OPS = {"BRA", "BRX", "JMP", "JMX", "BSSY", "BSYNC", "WARPSYNC", "BAR", "EXIT", "CALL", "RET", "BREAK", "BPT",
               "YIELD", "ENDCOLLECTIVE", "WARPGROUP"}
NO_DEST_OPS = {"STS", "STG", "STL", "ST", "RED", "CCTL", "MEMBAR", "NOP", "DEPBAR", "ERRBAR", "FENCE"} | BARRIER_OPS
FP64_OPS = {"DFMA", "DADD", "DMUL", "DSETP", "DMNMX"}

# phases of a round, in the order of the S2_PH counters of a -DDSP_PHASES build (the exit vote sits between refill and pass 1)
PHASES = ["check", "refill", "exit vote", "pass 1", "factor + pred. solve", "pass 2", "pass 3 + corr. solve", "pass 4", "pass 5"]
MARKERS = [("check", "convergence check"), ("refill", "(re)fill groups"), ("pass 1", "neighbours of the lane's block"),
           ("factor + pred. solve", "factorisation + predictor solve"), ("pass 2", "pass 2: predictor direction"),
           ("pass 3 + corr. solve", "pass 3: corrector right-hand side"), ("pass 4", "pass 4: corrector direction"),
           ("pass 5", "pass 5: step")]


def phase_lines(src: Path):
    """[(first line, phase)] of warp_body's round, and the line range of warp_body."""
    lines = src.read_text().splitlines()
    bounds = []
    body0 = next(i for i, s in enumerate(lines, 1) if "__device__ void warp_body(" in s)
    body1 = next(i for i, s in enumerate(lines, 1) if i > body0 and s.startswith("}"))
    for name, tag in MARKERS:
        hit = [i for i, s in enumerate(lines, 1) if "// ====" in s and s.rstrip().endswith(tag) and body0 < i < body1]
        if len(hit) != 1:
            raise SystemExit(f"phase marker '{tag}' found {len(hit)} times in {src.name}")
        bounds.append((hit[0], name))
    vote = [i for i, s in enumerate(lines, 1) if "if (cta_all(mode == 3))" in s and body0 < i < body1]
    if len(vote) != 1:
        raise SystemExit("exit vote not found")
    bounds.append((vote[0], "exit vote"))
    bounds.sort()
    return bounds, (body0, body1)


def phase_of(line, bounds):
    ph = None
    for first, name in bounds:
        if line >= first:
            ph = name
    return ph or "setup"


# ---------------------------------------------------------------------------------------------------- SASS
def run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(" ".join(map(str, cmd)) + "\n" + r.stdout + r.stderr)
    return r.stdout


def cuda_tool(name):
    p = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not os.path.exists(p):
        raise SystemExit(f"{name} not found")
    return p


def compile_cubin(tmp: Path, defines):
    out = tmp / "dsp_lp.cubin"
    run([cuda_tool("nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-cubin",
         f"-I{ROOT / 'include'}", *[f"-D{d}" for d in defines], str(CSRC / "dsp_lp.cu"), "-o", str(out)])
    return [out]


def kernel_sass(cubins, L, P):
    """(function name, nvdisasm -gi text of that function) of dsp_ipm_stage2_wb_kernel<L, P>."""
    tag = f"dsp_ipm_stage2_wb_kernelILi{L}ELi{P}E"
    for cb in cubins:
        text = run([cuda_tool("nvdisasm"), "-gi", str(cb)])
        out, name, on = [], None, False
        for s in text.splitlines():
            if s.startswith(".text."):
                on = tag in s
                if on:
                    name = s[len(".text."):].rstrip(":")
                continue
            if on:
                out.append(s)
        if out:
            return name, out
    raise SystemExit(f"no SASS for {tag} (built with -lineinfo for sm_90a?)")


INSN = re.compile(r"^\s*/\*([0-9a-f]+)\*/\s+(.*?)\s*;")
LINEINFO = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
REG = re.compile(r"(?<![\w.])(!?)(R\d+|RZ|P\d|PT|UR\d+|URZ|UP\d|UPT)(\.64)?(?![\w])")


def split_operands(rest):
    ops, depth, cur = [], 0, ""
    for ch in rest:
        if ch in "[{(":
            depth += 1
        elif ch in "]})":
            depth -= 1
        if ch == "," and depth == 0:
            ops.append(cur.strip()); cur = ""
        else:
            cur += ch
    if cur.strip():
        ops.append(cur.strip())
    return ops


def width_of(op, mods, role):
    """32-bit registers an R operand spans: 'dest' or 'src' role."""
    if op in FP64_OPS:
        return 2
    if op in ("F2F", "I2F", "F2I"):
        ts = [m for m in mods if re.fullmatch(r"[FSU](16|32|64)", m)]
        if len(ts) >= 2:
            return 2 if (ts[0] if role == "dest" else ts[1]).endswith("64") else 1
        if len(ts) == 1:
            return 2 if ts[0].endswith("64") else 1
        return 1
    if op == "CS2R":
        return 2
    for w, n in (("128", 4), ("64", 2)):
        if w in mods and op in ("LDS", "LDG", "LDL", "LD", "LDC", "STS", "STG", "STL", "ST", "ULDC", "SHFL", "ATOMG", "ATOMS", "RED"):
            return n
    return 1


def regs_of(operand, w):
    """32-bit general, uniform and predicate registers an operand names (RZ / PT excluded)"""
    out = []
    for neg, r, wide in REG.findall(operand):
        if r in ("RZ", "PT", "URZ", "UPT"):
            continue
        if r[0] == "R" or r.startswith("UR"):
            base = int(r[2:] if r.startswith("UR") else r[1:])
            pre = "UR" if r.startswith("UR") else "R"
            n = 2 if wide else w
            out += [f"{pre}{base + k}" for k in range(n)]
        else:
            out.append(r)
    return out


class Insn:                  # one SASS instruction: t = model finish time, pred = the instruction it waited for last
    __slots__ = ("addr", "text", "op", "line", "phase", "dst", "src", "lat", "barrier", "t", "pred")


def parse(lines, bounds, body):
    insns, line = [], None
    pending = []
    for s in lines:
        m = LINEINFO.search(s)
        if m:
            pending.append(m)
            continue
        mi = INSN.match(s)
        if not mi:
            continue
        if pending:
            # the frame of warp_body: the innermost location in dsp_stage2.cuh's warp_body lines that is not itself inlined
            # into another line of dsp_stage2.cuh, i.e. the line of the round the instruction belongs to
            cand = [int(x.group(2)) for x in pending
                    if x.group(1).endswith("dsp_stage2.cuh") and body[0] <= int(x.group(2)) <= body[1]
                    and (x.group(3) is None or not x.group(3).endswith("dsp_stage2.cuh"))]
            line = cand[0] if cand else -1
            pending = []
        ins = Insn()
        ins.addr = int(mi.group(1), 16)
        ins.text = mi.group(2)
        ins.line = line if line is not None else -1
        ins.phase = phase_of(ins.line, bounds) if ins.line and ins.line > 0 else "setup"
        body_txt = ins.text
        guard = []
        gm = re.match(r"^@(!?)(U?P\d|U?PT)\s+(.*)$", body_txt)
        if gm:
            if gm.group(2) not in ("PT", "UPT"):
                guard = [gm.group(2)]
            body_txt = gm.group(3)
        parts = body_txt.split(None, 1)
        full = parts[0]
        rest = parts[1] if len(parts) > 1 else ""
        op, *mods = full.split(".")
        ins.op = op
        ins.lat = LATENCY.get(op, DEFAULT_LATENCY)
        ins.barrier = op in BARRIER_OPS
        ops = split_operands(rest)
        dst, src = [], list(guard)
        if op in NO_DEST_OPS or not ops:
            for o in ops:
                src += regs_of(o, width_of(op, mods, "src"))
        else:
            nd = 1
            if "SETP" in op or op in ("SHFL", "PLOP3"):
                nd = 2
            else:                                        # carry-out predicates right after the destination
                while nd < len(ops) and re.fullmatch(r"U?P\d|U?PT", ops[nd]):
                    nd += 1
            for o in ops[:nd]:
                dst += regs_of(o, width_of(op, mods, "dest"))
            for o in ops[nd:]:
                src += regs_of(o, width_of(op, mods, "src"))
        ins.dst, ins.src = dst, src
        insns.append(ins)
    return insns


def analyse(insns):
    """longest weighted path of every phase; sets ins.t (finish time) and ins.pred (critical predecessor)."""
    res = {}
    for ph in ["setup"] + PHASES:
        seq = [i for i in insns if i.phase == ph]
        ready, writer = {}, {}
        floor, floor_src, tmax, tmax_src = 0, None, 0, None
        for ins in seq:
            start, pred = floor, floor_src
            for r in ins.src:
                if ready.get(r, 0) > start:
                    start, pred = ready[r], writer[r]
            ins.t = start + (0 if ins.barrier else ins.lat)
            ins.pred = pred
            if ins.barrier:
                ins.t = max(start, tmax)
                ins.pred = tmax_src if tmax > start else pred
                floor, floor_src = ins.t, ins
            for r in ins.dst:
                ready[r], writer[r] = ins.t, ins
            if ins.t > tmax:
                tmax, tmax_src = ins.t, ins
        res[ph] = dict(
            insns=len(seq),
            fp64=sum(i.op in FP64_OPS for i in seq),
            shfl=sum(i.op == "SHFL" for i in seq),
            lds=sum(i.op == "LDS" for i in seq),
            mufu=sum(i.op == "MUFU" for i in seq),
            branches=sum(i.barrier for i in seq),
            path=tmax,
            end=tmax_src,
        )
    return res


def chain(end):
    out = []
    while end is not None:
        out.append(end)
        end = end.pred
    return out[::-1]


def compress(ch):
    """consecutive runs of one source line: (line, instructions, model cycles, opcodes)"""
    out = []
    prev_t = 0
    for i in ch:
        dt = i.t - prev_t
        prev_t = i.t
        if out and out[-1][0] == i.line:
            out[-1][1] += 1; out[-1][2] += dt; out[-1][3].add(i.op)
        else:
            out.append([i.line, 1, dt, {i.op}])
    return out


def longest_chains(insns, n):
    """the n longest chains, each sharing at most half of its instructions with a longer one already listed: chains end in
    sinks (results no later instruction of the phase reads)"""
    used = set()
    for i in insns:
        if i.pred is not None:
            used.add(id(i.pred))
    sinks = sorted((i for i in insns if id(i) not in used and i.phase in PHASES and not i.barrier), key=lambda i: -i.t)
    out, taken = [], []
    for s in sinks:
        ch = chain(s)
        ids = {id(i) for i in ch}
        if any(len(ids & t) * 2 > len(ids) for t in taken):
            continue
        taken.append(ids)
        out.append((s, ch))
        if len(out) == n:
            break
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--kernel", default="8,3", help="L,P of the instantiation (default 8,3)")
    ap.add_argument("--lib", default=str(CSRC / "libdsp_lp.so"))
    ap.add_argument("--cubin")
    ap.add_argument("--compile", action="store_true", help="compile dsp_lp.cu (-lineinfo, sm_90a) into a temporary directory")
    ap.add_argument("-D", dest="defines", action="append", default=[], help="extra macro for --compile")
    ap.add_argument("--chains", type=int, default=10)
    ap.add_argument("--json", help="write the per-phase table as JSON")
    a = ap.parse_args(argv)
    L, P = map(int, a.kernel.split(","))
    bounds, body = phase_lines(STAGE2)
    with tempfile.TemporaryDirectory() as td:
        td = Path(td)
        if a.cubin:
            cubins = [Path(a.cubin)]
        elif a.compile:
            cubins = compile_cubin(td, a.defines)
        else:
            lib = Path(a.lib).resolve()
            if not lib.exists():
                raise SystemExit(f"{lib} not built (python -m dispatches_b200.csrc.build)")
            subprocess.run([cuda_tool("cuobjdump"), "-xelf", "all", str(lib)], cwd=td, capture_output=True, check=True)
            cubins = sorted(td.glob("*.cubin"))
        name, lines = kernel_sass(cubins, L, P)
    insns = parse(lines, bounds, body)
    res = analyse(insns)
    print(f"dsp_ipm_stage2_wb_kernel<{L},{P}>: {len(insns)} SASS instructions, {sum(i.op in FP64_OPS for i in insns)} FP64")
    print("MODEL (not measured): longest dependent path per phase, latencies "
          + ", ".join(f"{k} {v}" for k, v in LATENCY.items()) + f", other {DEFAULT_LATENCY}; branches are barriers")
    print(f"{'phase':<22}{'insns':>7}{'FP64':>6}{'SHFL':>6}{'LDS':>5}{'MUFU':>6}{'branch':>8}{'path (model cyc)':>18}")
    tot = 0
    for ph in PHASES:
        r = res[ph]
        tot += r["path"]
        print(f"{ph:<22}{r['insns']:>7}{r['fp64']:>6}{r['shfl']:>6}{r['lds']:>5}{r['mufu']:>6}{r['branches']:>8}{r['path']:>18}")
    print(f"{'round (sum)':<22}{sum(res[p]['insns'] for p in PHASES):>7}{sum(res[p]['fp64'] for p in PHASES):>6}"
          f"{sum(res[p]['shfl'] for p in PHASES):>6}{sum(res[p]['lds'] for p in PHASES):>5}{sum(res[p]['mufu'] for p in PHASES):>6}"
          f"{sum(res[p]['branches'] for p in PHASES):>8}{tot:>18}")
    print(f"(outside the round's phases: {res['setup']['insns']} instructions)")
    print(f"\nthe {a.chains} longest chains (model cycles), by source line of {STAGE2.name}: line(cycles) over runs of one line")
    for k, (s, ch) in enumerate(longest_chains(insns, a.chains)):
        segs = compress(ch)
        print(f"{k + 1:>2}. {s.phase}: {s.t} cycles, {len(ch)} instructions, ends at line {s.line} ({s.op})")
        print("    " + " ".join(f"{ln}({c})" for ln, n, c, ops in segs))
    if a.json:
        Path(a.json).write_text(json.dumps({"kernel": f"{L},{P}", "model_latency": LATENCY, "default_latency": DEFAULT_LATENCY,
                                            "phases": {p: {k: v for k, v in res[p].items() if k != "end"} for p in PHASES}},
                                           indent=1))
    return res


if __name__ == "__main__":
    main()
