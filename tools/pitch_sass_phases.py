"""Static SASS of pitch_kernel per phase (no GPU needed): the issue-side half of tools/pitch_phase_profile.py's account.

    python tools/pitch_sass_phases.py [path/to/lib.so or pitch.cu.o] [path/to/the pitch.cu it was built from]

Every instruction is attributed to the kernel-body source line it comes from (the outermost call site of inlined helpers,
from the line table that -lineinfo puts in the cubin), and a line to the phase whose trace point PT(k) is the first at or
below it -- the same phases as the clock trace.  Per phase: instructions, FP32 arithmetic (FFMA/FADD/FMUL/FMNMX),
shared-memory loads and stores, and each loop body (a backward branch) with its size, which times the loop's trip count
from the source gives that loop's issue per warp.  Static counts: a loop body is counted once.
"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "nnnoiseless_b200", "lib", "libnnnoiseless_b200.so")
SRC = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "nnnoiseless_b200", "csrc", "pitch.cu")
NAMES = {0: "prologue", 1: "Ph1 downsample", 3: "Ph2 autocorr", 5: "Ph3 LPC", 7: "Ph4 FIR", 9: "Ph5 coarse FMA | chains", 11: "Ph6a select",
         13: "Ph6x exact coarse", 15: "Ph6b fine windows | Ph7 | yy_lookup", 17: "Ph8 fine select + lags", 19: "Ph9 rd FMA",
         20: "Ph10g ladder gains", 21: "Ph10a ladder", 23: "Ph10x exact ladder", 24: "Ph11 lane-tasks", 26: "Ph11 final"}


def phase_map():
    src = open(SRC).read().split("\n")
    k0 = next(i for i, l in enumerate(src, 1) if "pitch_kernel(const float*" in l)
    k1 = next(i for i, l in enumerate(src, 1) if i > k0 and l.startswith("}"))
    points = [(i, int(m.group(1))) for i, l in enumerate(src, 1) if k0 <= i <= k1 for m in [re.match(r"\s*PT\((\d+)\);", l)] if m]
    return k0, k1, points


def main():
    k0, k1, points = phase_map()
    with tempfile.TemporaryDirectory() as d:
        subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(LIB)], cwd=d, capture_output=True, check=True)
        cub = os.path.join(d, next(f for f in os.listdir(d) if f.startswith("pitch") and f.endswith(".cubin")))
        sass = subprocess.run(["nvdisasm", "-gi", "-c", cub], capture_output=True, text=True, check=True).stdout
    start = re.search(r"\n\.text\.\S*pitch_kernel\S*:", sass).start()
    end = sass.find("\n//----", start + 1)
    body = sass[start:end if end > 0 else len(sass)]
    line, insts = None, []  # (phase, opcode, branch target label)
    labels = {}
    for l in body.split("\n"):
        m = re.match(r"\s*//## File (.*)", l)
        if m:
            locs = re.findall(r'"([^"]+)", line (\d+)', m.group(1))
            f, n = locs[-1]
            n = int(n)
            line = n if os.path.basename(f) == os.path.basename(SRC) and k0 <= n <= k1 else None
            continue
        m = re.match(r"(\.L_x_\d+):", l.strip())
        if m:
            labels[m.group(1)] = len(insts)
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)(.*)", l)
        if not m:
            continue
        ph = "subroutines (div/sqrt slow paths)" if line is None else \
            NAMES.get(next((k for i, k in points if i >= line), 26), "?")
        tgt = re.search(r"`\((\.L_x_\d+)\)", m.group(4))
        insts.append((ph, m.group(3), tgt.group(1) if tgt else None))
    per = collections.OrderedDict()
    for ph, op, _ in insts:
        c = per.setdefault(ph, collections.Counter())
        c["all"] += 1
        base = op.split(".")[0]
        if base in ("FFMA", "FADD", "FMUL", "FMNMX"):
            c["fp32"] += 1
        elif base in ("LDS", "STS"):
            c[base] += 1
    print("pitch_kernel static SASS per phase (%s)" % os.path.basename(LIB))
    print("%-36s %6s %6s %5s %5s" % ("phase", "instr", "fp32", "LDS", "STS"))
    for ph, c in per.items():
        print("%-36s %6d %6d %5d %5d" % (ph, c["all"], c["fp32"], c["LDS"], c["STS"]))
    print("\nloop bodies (backward branches): phase, instructions in the body, of them fp32 / LDS")
    for j, (ph, op, tgt) in enumerate(insts):
        if op.startswith("BRA") and tgt in labels and labels[tgt] <= j:
            b = insts[labels[tgt]:j + 1]
            if any(x[0] != ph for x in b):
                continue  # a loop around several phases (the rounds of Ph6x, the stream queue of Ph9)
            nfp = sum(1 for x in b if x[1].split(".")[0] in ("FFMA", "FADD", "FMUL", "FMNMX"))
            nl = sum(1 for x in b if x[1].startswith("LDS"))
            print("  %-36s %5d  %4d / %3d" % (ph, len(b), nfp, nl))


if __name__ == "__main__":
    main()
