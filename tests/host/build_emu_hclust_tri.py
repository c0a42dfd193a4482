#!/usr/bin/env python
"""TEST INFRASTRUCTURE: the host-emulation build of tests/host/build_emu_subclusters.py plus the packed-triangle linkage
(icnv_hclust_tri.cu), into a directory of the caller's choosing (tests/test_hclust_tri_emulated.py uses a temporary one).
The sources go through build_emu.transform() unchanged and are compiled with the same flags.  icnv_hclust_tri.cu gets the
stand-ins icnv_subclusters.cu gets (the stream-ordered allocator, a fixed 4 GB free, timing events with zero elapsed time).

    python tests/host/build_emu_hclust_tri.py OUT_DIR     -> OUT_DIR/libinfercnv_b200_emu_hclust_tri.so
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

SOURCES = build_emu_subclusters.SOURCES + ["icnv_hclust_tri.cu"]
STANDINS = dict(build_emu_subclusters.STANDINS,
                **{"icnv_hclust_tri.cu": build_emu_subclusters.STANDINS["icnv_subclusters.cu"]})


def build(out_dir: str) -> str:
    gen = os.path.join(out_dir, "src")
    os.makedirs(gen, exist_ok=True)
    files = []
    for f in SOURCES:
        text, n = build_emu.transform(open(os.path.join(build_emu.CSRC, f)).read())
        assert "<<<" not in text, f"{f}: a launch was not recognised"
        if f in STANDINS:
            inc = '#include "icnv_common.cuh"\n'
            assert inc in text
            text = text.replace(inc, inc + STANDINS[f], 1)
        dst = os.path.join(gen, f.replace(".cu", ".emu.cpp"))
        open(dst, "w").write(f"// generated from infercnv_b200/csrc/{f} ({n} launches rewritten)\n" + text)
        files.append(dst)
    out = os.path.join(out_dir, "libinfercnv_b200_emu_hclust_tri.so")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    cmd = [gxx, "-O1", "-std=c++17", "-fPIC", "-shared", "-D__CUDACC__", "-DICNV_EMU", "-Wall", "-Wno-unknown-pragmas",
           "-Wno-attributes", "-Wno-unused-function", "-Wno-unused-variable", "-Wno-unused-but-set-variable", "-mfma",
           "-ffp-contract=off", "-pthread", "-rdynamic", "-fno-omit-frame-pointer", "-I", os.path.join(HERE, "emu"),
           "-I", build_emu.CSRC, "-o", out, *files]
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    print(build(sys.argv[1]))
