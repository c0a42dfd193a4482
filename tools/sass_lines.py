#!/usr/bin/env python
"""Static SASS census of one kernel, by source line (no GPU needed).

    python tools/sass_lines.py icnv_smooth.cu cell_pipeline3_kernelILi1024 [--lines A:B] [--ops]

Compiles csrc/<file> to a cubin for sm_90a with -lineinfo, disassembles it with `nvdisasm -g -c` and attributes
every instruction of the kernel whose mangled name contains the pattern to the source line of the preceding
line marker.  Prints instructions per source line (with the source text) and per opcode class: the instruction
count of a loop body is the number the issue-bound kernels (DESIGN.md K2 / K3) are tuned against before a GPU
run is spent on them.  --lines restricts the listing to a source range of the kernel's own file."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "infercnv_b200", "csrc")


def classify(op):
    if op.startswith(("DFMA", "DADD", "DMUL", "DSETP", "DMNMX")):
        return "fp64"
    if op.startswith(("F2F", "I2F", "F2I", "MUFU", "FRND")):
        return "convert/sfu"
    if op.startswith(("FFMA", "FADD", "FMUL", "FSETP", "FSEL", "FMNMX")):
        return "fp32"
    if op.startswith(("LDS", "STS", "ATOMS", "LDSM")):
        return "shared"
    if op.startswith(("LDG", "STG", "LD.", "ST.", "ATOMG", "RED", "LDL", "STL", "UBLKCP", "LDGSTS", "LDC")):
        return "global/local/const"
    if op.startswith(("BAR", "SYNCS", "WARPSYNC", "BSSY", "BSYNC", "BRA", "EXIT", "CALL", "RET", "NANOSLEEP", "DEPBAR", "ERRBAR")):
        return "control/barrier"
    if op.startswith(("SHFL", "VOTE", "REDUX", "MATCH")):
        return "warp"
    return "int/move/select"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("source")
    ap.add_argument("pattern")
    ap.add_argument("--lines", default=None)
    ap.add_argument("--ops", action="store_true", help="opcode histogram per listed line")
    ap.add_argument("--loops", action="store_true", help="list the loops (backward branches): body length in instructions, "
                    "source lines it spans - the innermost ones are the per-gene costs quoted in DESIGN.md")
    a = ap.parse_args()
    src = os.path.join(CSRC, a.source)
    with tempfile.TemporaryDirectory() as td:
        cubin = os.path.join(td, "k.cubin")
        subprocess.check_call(["nvcc", "-ccbin", "/usr/bin/g++", "-O3", "-std=c++17", "-lineinfo", "-gencode",
                               "arch=compute_90a,code=sm_90a", "-cubin", src, "-o", cubin], stderr=subprocess.DEVNULL)
        dis = subprocess.run(["nvdisasm", "-g", "-c", cubin], capture_output=True, text=True).stdout
    text = open(src).read().split("\n")
    lo, hi = (int(v) for v in a.lines.split(":")) if a.lines else (0, 10 ** 9)
    insts = []      # (address, opcode, source line or None, label in front or None, branch target label or None)
    pending_label = None
    per_line = collections.Counter()
    per_line_ops = collections.defaultdict(collections.Counter)
    classes = collections.Counter()
    other_files = collections.Counter()
    inside, cur = False, None
    for ln in dis.split("\n"):
        if ln.startswith(".text."):
            inside = a.pattern in ln
            cur = None
            continue
        if ln.startswith("//-----"):
            inside = False
            continue
        if not inside:
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = (os.path.basename(m[1]), int(m[2]))
            continue
        m = re.match(r"(\.L_x_\d+):", ln)
        if m:
            pending_label = m[1]
            continue
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)(.*)", ln)
        if m:
            tgt = re.search(r"`\((\.L_x_\d+)\)", m[3])
            insts.append((int(m[1], 16), m[2], cur[1] if cur and cur[0] == os.path.basename(src) else None, pending_label,
                          tgt[1] if tgt and m[2].startswith("BRA") else None))
            pending_label = None
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
        if not m or cur is None:
            continue
        op = m[1]
        if cur[0] == os.path.basename(src):
            if lo <= cur[1] <= hi:
                per_line[cur[1]] += 1
                per_line_ops[cur[1]][op.split(".")[0]] += 1
                classes[classify(op)] += 1
        else:
            other_files[cur[0]] += 1
            if a.lines is None:
                classes[classify(op)] += 1
    if a.loops:
        at = {lab: i for i, (_, _, _, lab, _) in enumerate(insts) if lab}
        print(f"# loops of {a.pattern} (backward branches): instructions in the body, source lines spanned, body opcode classes")
        for i, (addr, op, line, lab, tgt) in enumerate(insts):
            if tgt and tgt in at and at[tgt] <= i:
                body = insts[at[tgt]:i + 1]
                lines = [b[2] for b in body if b[2]]
                if a.lines and not (lines and lo <= min(lines) and max(lines) <= hi):
                    continue
                cls = collections.Counter(classify(b[1]) for b in body)
                calls = sum(1 for b in body if b[1].startswith("CALL"))
                print(f"{len(body):5d} instr  lines {min(lines) if lines else '?'}-{max(lines) if lines else '?'}  "
                      f"{dict(cls.most_common())}" + (f"  (contains {calls} out-of-line calls: slow paths)" if calls else ""))
        return 0
    total = sum(per_line.values())
    print(f"# {a.pattern}: {total} instructions attributed to {os.path.basename(src)}"
          + (f" lines {lo}-{hi}" if a.lines else "") + f"; inlined headers: {dict(other_files)}")
    for line in sorted(per_line):
        ops = ("  [" + " ".join(f"{k}:{v}" for k, v in per_line_ops[line].most_common()) + "]") if a.ops else ""
        print(f"{line:5d} {per_line[line]:5d}  {text[line - 1].strip()[:110]}{ops}")
    print("# classes:", dict(classes.most_common()))


if __name__ == "__main__":
    sys.exit(main())
