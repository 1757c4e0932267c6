"""Register account of analysis_warp_kernel (no GPU needed): what its persistent loop keeps live, phase by phase.

    python tools/analysis_regs.py [--blocks 3,4,5] [--base REV]

Compiles nnnoiseless_b200/csrc/spectral_warp.cu for sm_90a with the library's flags, once per blocks-per-SM count N
(-DNNB_ANALYSIS_BLOCKS=N, i.e. __launch_bounds__(128, N)), in a temporary directory.  For every analysis_warp_kernel
instantiation it prints a table with one column per build:
  - registers and spill bytes, from ptxas -v;
  - per loop phase, the peak number of live registers over the phase's instructions (nvdisasm --print-life-ranges).
    An instruction belongs to the phase of the kernel-body source line it comes from (the outermost frame of the
    -lineinfo line table; inside fft480_warp, the line of that function);
  - the registers live into the kernel's first instruction: values that some path reads before any write.  Each is
    listed under the phase that first writes it.  A write under a predicate does not end a live range, so values
    loaded on both arms of an if-converted branch (the staging read's even / odd pitch loads) are counted too;
and then every spill store and reload (STL / LDL) with the phase and the innermost source line it comes from.
With --base REV the same source tree at git revision REV (its csrc and include directories) is compiled too, side by
side, and the synthesis kernels' SASS (encodings included) is compared between the two.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nnnoiseless_b200.build import ARCH, COMMON, NVCC  # noqa: E402  the library's own flags

SRC_REL = os.path.join("nnnoiseless_b200", "csrc", "spectral_warp.cu")
INST = {"ILb0ELb0E": "<false,false>", "ILb1ELb0E": "<true,false>", "ILb1ELb1E": "<true,true>"}
# (phase, regex of its first source line), in source order; a line belongs to the last phase starting at or above it
KERNEL_PHASES = [("prologue", r"analysis_warp_kernel\(BatchBuffers"), ("loop head, mbarrier wait", r"for \(int it = 0;"),
                 ("staging read", r"float2 vx\[15\], vp\[15\];"), ("fft480", r"fft480_warp<true>\("),
                 ("even/odd split", r"// even/odd split"), ("band sums", r"band_sums_warp<3>\("),
                 ("issue next stream", r"fence_proxy_async\(\);"), ("feature tail", r"// ---- features")]
FFT_PHASES = [("fft480: dft15 x2", r"dft15\(vx\);"), ("fft480: twiddle, transpose stores", r"for \(int k1 = 1;"),
              ("fft480: fft32 loads + butterflies", r"float2 r\[32\];"), ("fft480: fft32 stores", r"const int base =")]
PHASE_ORDER = [p for p, _ in KERNEL_PHASES[:3]] + ["fft480: call site"] + [p for p, _ in FFT_PHASES] + [p for p, _ in KERNEL_PHASES[4:]] + ["subroutines"]


def run(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    if r.returncode != 0:
        sys.exit("failed: %s\n%s%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r


def body_range(src, head):
    """(first, last) 1-based lines of the function whose signature line matches head."""
    k0 = next(i for i, l in enumerate(src, 1) if re.search(head, l))
    k1 = next(i for i, l in enumerate(src, 1) if i > k0 and l.startswith("}"))
    return k0, k1


def phase_starts(src, lo, hi, phases):
    out, at = [], lo
    for name, rx in phases:
        at = next((i for i in range(at, hi + 1) if re.search(rx, src[i - 1])), None)
        if at is None:
            sys.exit("phase marker %r not found in %s" % (rx, SRC_REL))
        out.append((at, name))
    return out


def phase_of(starts, line):
    return [name for at, name in starts if at <= line][-1]


def compile_tree(tree, blocks, d):
    """cubin and ptxas log of tree's spectral_warp.cu at the given blocks per SM."""
    src = os.path.join(tree, SRC_REL)
    text = open(src).read()
    if "NNB_ANALYSIS_BLOCKS" not in text:  # a revision from before the knob (an extracted copy): the constant is set in place
        assert tree != ROOT
        open(src, "w").write(re.sub(r"constexpr int ANALYSIS_BLOCKS = \d+;", "constexpr int ANALYSIS_BLOCKS = NNB_ANALYSIS_BLOCKS;", text))
    cub = os.path.join(d, "sw_%d.cubin" % blocks)
    r = run([NVCC] + ARCH + COMMON + ["-DNNB_ANALYSIS_BLOCKS=%d" % blocks, "-cubin", src, "-o", cub])
    return cub, r.stderr, src


def ptxas_info(log):
    """mangled name -> (registers, spill stores, spill loads)"""
    out, cur, spill = {}, None, (0, 0)
    for l in log.split("\n"):
        m = re.search(r"Compiling entry function '(\S+)'", l)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
        if m:
            spill = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", l)
        if m and cur:
            out[cur] = (int(m.group(1)),) + spill
            cur = None
    return out


def sections(text):
    """kernel name -> its lines, for the analysis and synthesis kernels of an nvdisasm listing"""
    out, name = {}, None
    for l in text.split("\n"):
        m = re.match(r"//-+ \.text\.(\S+) -+", l.strip())
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            out[name].append(l)
    return out


def account(tree, blocks, d):
    cub, log, src_path = compile_tree(tree, blocks, d)
    src = open(src_path).read().split("\n")
    k0, k1 = body_range(src, r"analysis_warp_kernel\(BatchBuffers")
    f0, f1 = body_range(src, r"void fft480_warp\(")
    kstarts = phase_starts(src, k0, k1, KERNEL_PHASES)
    fstarts = phase_starts(src, f0, f1, FFT_PHASES)
    fft_call = next(at for at, name in kstarts if name == "fft480")
    base = os.path.basename(src_path)
    info = ptxas_info(log)
    gi = sections(run(["nvdisasm", "-c", "-gi", cub]).stdout)
    plr = sections(run(["nvdisasm", "-c", "-plr", cub]).stdout)
    res = {}
    for name in gi:
        tag = next((v for k, v in INST.items() if "analysis_warp_kernel" + k in name), None)
        if tag is None:
            continue
        # phase and innermost source line of every instruction, by address
        phase, inner, ph = {}, {}, "subroutines"
        chain, fresh = [], False
        for l in gi[name]:
            m = re.match(r"\s*//## File (.*)", l)
            if m:
                if not fresh:
                    chain, fresh = [], True
                f, n = re.findall(r'"([^"]+)", line (\d+)', m.group(1))[0]
                chain.append((os.path.basename(f), int(n)))
                continue
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/", l)
            if not m:
                continue
            if fresh:
                fresh = False
                outer = chain[-1] if chain else None
                ph = "subroutines"
                if outer and outer[0] == base and k0 <= outer[1] <= k1:
                    ph = phase_of(kstarts, outer[1])
                    if outer[1] == fft_call:
                        fl = next((n for f, n in chain if f == base and f0 <= n <= f1), None)
                        ph = phase_of(fstarts, fl) if fl else "fft480: call site"
                in_line = "%s:%d" % chain[0] if chain else "?"
            a = int(m.group(1), 16)
            phase[a], inner[a] = ph, (in_line, l.split("*/", 1)[1].strip())
        # live GPRs per instruction, and the registers live into the first one
        lines = plr[name]
        hdr = next(l for l in lines if re.search(r"//\s*\|\s+#\s+0 1 2", l))
        h = hdr[hdr.rindex("// |") + 3:]
        gseg = h.split("|")[1]
        cols = [(m.end(), int(m.group(1))) for m in re.finditer(r"(\d+)", gseg)]  # a register's mark: under its label's last digit
        peak, entry, first_def = collections.Counter(), None, {}
        for l in lines:
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/", l)
            if not m or "// |" not in l:
                continue
            a = int(m.group(1), 16)
            row = l[l.rindex("// |") + 3:]
            cnt = int(row.split("|")[1].split()[0]) if row.split("|")[1].split() else 0
            p = phase.get(a, "subroutines")
            peak[p] = max(peak[p], cnt)
            if entry is None:
                entry = [r for c, r in cols if c < len(row) and row[c] == ":"]
            for c, r in cols:
                if c < len(row) and row[c] in "^x" and r not in first_def:
                    first_def[r] = p
        ent = collections.Counter(first_def.get(r, "never written") for r in entry)
        spills = collections.Counter((phase[a], inner[a][0], inner[a][1].split()[0] if not inner[a][1].startswith("@") else inner[a][1].split()[1])
                                     for a in phase if re.search(r"\b(STL|LDL)\b", inner[a][1]))
        regs, st, ld = next(v for k, v in info.items() if k in name)
        res[tag] = dict(regs=regs, spill_st=st, spill_ld=ld, peak=peak, entry=len(entry), entry_by=ent, spills=spills)
    return res, cub


def synthesis_sass(cub):
    t = run(["cuobjdump", "-sass", cub]).stdout
    t = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_spectral_warp_cu_[0-9a-f]+", "ANON", t)  # the anonymous namespace's per-build hash
    t = re.sub(r"[ \t]+", " ", t)
    return {p.split("\n", 1)[0].strip(): p for p in re.split(r"\n\s*Function : ", t)[1:] if "synthesis_warp_kernel" in p.split("\n", 1)[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", default="3,4,5", help="blocks per SM to compile for, comma-separated")
    ap.add_argument("--base", default="", help="also account the source at this git revision")
    a = ap.parse_args()
    blocks = [int(b) for b in a.blocks.split(",")]
    with tempfile.TemporaryDirectory() as d:
        trees = [("tree", ROOT)]
        if a.base:
            bt = os.path.join(d, "base")
            os.makedirs(bt)
            arch = subprocess.run(["git", "-C", ROOT, "archive", a.base, "nnnoiseless_b200/csrc", "include"], capture_output=True, check=True).stdout
            subprocess.run(["tar", "-x", "-C", bt], input=arch, check=True)
            trees.insert(0, ("base " + a.base, bt))
        cols, cubs = [], {}
        for label, tree in trees:
            for b in blocks:
                od = os.path.join(d, "%s_%d" % (label.split()[0], b))
                os.makedirs(od)
                res, cub = account(tree, b, od)
                cols.append(("%s (128, %d)" % (label, b), res))
                cubs.setdefault(label, cub)
        w = max(22, max(len(c) for c, _ in cols) + 1)
        for tag in INST.values():
            print("\nanalysis_warp_kernel%s" % tag)
            print("%-46s" % "" + "".join("%*s" % (w, c) for c, _ in cols))
            rows = [("registers", lambda r: r["regs"]), ("spill stores / loads, bytes", lambda r: "%d / %d" % (r["spill_st"], r["spill_ld"]))]
            rows += [("peak live: " + p, (lambda p: lambda r: r["peak"].get(p, "-"))(p)) for p in PHASE_ORDER]
            rows += [("live into the first instruction", lambda r: r["entry"])]
            for name, f in rows:
                if all(f(res[tag]) == "-" for _, res in cols):
                    continue
                print("%-46s" % name + "".join("%*s" % (w, f(res[tag])) for _, res in cols))
            for c, res in cols:
                r = res[tag]
                if r["entry"]:
                    print("  %s: the %d registers live into the first instruction, by the phase that first writes them: %s" %
                          (c, r["entry"], ", ".join("%s %d" % kv for kv in r["entry_by"].most_common())))
                if r["spills"]:
                    print("  %s: spill sites (phase, innermost source line, opcode: count)" % c)
                    for (p, line, op), n in sorted(r["spills"].items()):
                        print("    %-34s %-22s %-6s %3d" % (p, line, op, n))
        if a.base:
            s0, s1 = synthesis_sass(cubs[trees[0][0]]), synthesis_sass(cubs["tree"])
            same = sorted(s0) == sorted(s1) and all(s0[k] == s1[k] for k in s0)
            print("\nsynthesis_warp_kernel SASS, %d instantiations: %s" % (len(s0), "identical to the base" if same else "DIFFERENT from the base"))


if __name__ == "__main__":
    main()
