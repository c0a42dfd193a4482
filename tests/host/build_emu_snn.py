#!/usr/bin/env python
"""TEST INFRASTRUCTURE: the host-emulation build of tests/host/build_emu_subclusters.py plus the SNN kernels (icnv_snn.cu),
into a directory of the caller's choosing (tests/test_snn_emulated_and_r.py uses a temporary one).  The sources go through
build_emu.transform() unchanged and are compiled with the same flags.  icnv_snn.cu gets the stand-ins icnv_subclusters.cu
gets (the stream-ordered allocator, a fixed 4 GB free, timing events with zero elapsed time) and one for its inline PTX:
the FP64 tensor-core product dmma_16x8x4 (mma.sync m16n8k4 .f64), rebuilt from the emulation's warp shuffles on the PTX
ISA's fragment layout - every lane publishes its A pair and B value, every lane forms its four D entries with one fma per
k in ascending k.

    python tests/host/build_emu_snn.py OUT_DIR     -> OUT_DIR/libinfercnv_b200_emu_snn.so
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_emu  # noqa: E402
import build_emu_subclusters  # noqa: E402

SOURCES = build_emu_subclusters.SOURCES + ["icnv_snn.cu"]
STANDINS = dict(build_emu_subclusters.STANDINS, **{"icnv_snn.cu": build_emu_subclusters.STANDINS["icnv_subclusters.cu"]})
# a0 = A[g][t], a1 = A[g + 8][t], b = B[t][g], d[i] = D[g + 8 (i / 2)][2 t + i % 2], g = lane / 4, t = lane % 4
DMMA = """{
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    double A[16][4], B[4][8];
    for (int l = 0; l < 32; ++l) {
        const double x0 = __shfl_sync(0xffffffffu, a0, l), x1 = __shfl_sync(0xffffffffu, a1, l), y = __shfl_sync(0xffffffffu, b, l);
        A[l >> 2][l & 3] = x0;
        A[(l >> 2) + 8][l & 3] = x1;
        B[l & 3][l >> 2] = y;
    }
    for (int i = 0; i < 4; ++i) {
        const int r = g + 8 * (i >> 1), c = 2 * t + (i & 1);
        double s = d[i];
        for (int kk = 0; kk < 4; ++kk) s = fma(A[r][kk], B[kk][c], s);
        d[i] = s;
    }
}"""


def build(out_dir: str) -> str:
    gen = os.path.join(out_dir, "src")
    os.makedirs(gen, exist_ok=True)
    files = []
    for f in SOURCES:
        text = open(os.path.join(build_emu.CSRC, f)).read()
        if f == "icnv_snn.cu":
            swapped = build_emu.replace_body(text, "dmma_16x8x4", DMMA)
            assert swapped != text, "dmma_16x8x4 not found"
            text = swapped
        text, n = build_emu.transform(text)
        assert "<<<" not in text, f"{f}: a launch was not recognised"
        if f in STANDINS:
            inc = '#include "icnv_common.cuh"\n'
            assert inc in text
            text = text.replace(inc, inc + STANDINS[f], 1)
        dst = os.path.join(gen, f.replace(".cu", ".emu.cpp"))
        open(dst, "w").write(f"// generated from infercnv_b200/csrc/{f} ({n} launches rewritten)\n" + text)
        files.append(dst)
    out = os.path.join(out_dir, "libinfercnv_b200_emu_snn.so")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    cmd = [gxx, "-O1", "-std=c++17", "-fPIC", "-shared", "-D__CUDACC__", "-DICNV_EMU", "-Wall", "-Wno-unknown-pragmas",
           "-Wno-attributes", "-Wno-unused-function", "-Wno-unused-variable", "-Wno-unused-but-set-variable", "-mfma",
           "-ffp-contract=off", "-pthread", "-rdynamic", "-fno-omit-frame-pointer", "-I", os.path.join(HERE, "emu"),
           "-I", build_emu.CSRC, "-o", out, *files]
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    print(build(sys.argv[1]))
