"""Build libinfercnv_b200.so in-tree with nvcc for sm_90a (no JIT cache: the .so is built once by
__graft_entry__.build() and loaded from the tree).  `python -m infercnv_b200.build [--force] [--verbose]`."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libinfercnv_b200.so")
SOURCES = ["icnv_api.cu", "icnv_smooth.cu", "icnv_viterbi.cu", "icnv_median_filter.cu", "icnv_reduce.cu",
           "icnv_synth.cu", "icnv_regions.cu", "icnv_ingest.cu", "icnv_dist.cu", "icnv_hclust.cu",
           "icnv_random_trees.cu", "icnv_de.cu", "icnv_de_multi.cu", "icnv_bayes.cu", "icnv_smooth_coords.cu",
           "icnv_subclusters.cu", "icnv_snn.cu", "icnv_hclust_tri.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libinfercnv_b200.so")


def _stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "infercnv_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return OUT
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    # the image's /opt/gcc wrapper lacks pieces; the distro g++ is the supported host compiler
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    common = [nvcc(), "-ccbin", ccbin, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-fvisibility=hidden",
              "-Xptxas", "-v" if verbose else "-warn-spills"]
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = common + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(f"--- {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    link = [nvcc(), "-ccbin", ccbin, "-shared", *ARCH, "-o", OUT, *objs, "-Xlinker", "-rpath=/usr/local/cuda/lib64"]
    subprocess.check_call(link)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
