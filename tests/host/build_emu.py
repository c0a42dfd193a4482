#!/usr/bin/env python
"""TEST INFRASTRUCTURE: build tests/host/_build/libinfercnv_b200_emu.so - the byte / index kernels of the library
(icnv_regions.cu, icnv_ingest.cu, icnv_reduce.cu) and the host entry points of icnv_api.cu compiled by g++ from the SAME
source text against the execution-model emulation in tests/host/emu/cuda_runtime.h.  The only transformation is
syntactic: `kernel<<<grid, block, smem, stream>>>(args);` becomes `EMU_LAUNCH(kernel, (grid, block, smem, stream), (args));`.
Dynamic shared memory declarations become pointers into the emulation's per-block buffer, and the handful of inline-PTX
wrappers (TMA bulk copy + mbarrier, cp.async) get synchronous stand-ins (PTX_STANDINS below).  FP contraction is off:
only the fma() calls written in the source fuse, as with nvcc's explicit intrinsics; where nvcc would contract a plain
a * b + c on its own the emulation rounds twice, which the parity tolerances absorb.

Used by tests/test_emulated_kernels.py only.  The package never loads this library."""
from __future__ import annotations

import os
import re
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "infercnv_b200", "csrc")
OUT_DIR = os.path.join(HERE, "_build")
OUT = os.path.join(OUT_DIR, "libinfercnv_b200_emu.so")
EMULATED = ["icnv_api.cu", "icnv_regions.cu", "icnv_ingest.cu", "icnv_reduce.cu", "icnv_smooth.cu", "icnv_viterbi.cu",
            "icnv_median_filter.cu", "icnv_synth.cu", "icnv_dist.cu"]

# The asynchronous-copy primitives (inline PTX) get synchronous stand-ins: the copy happens when it is issued - the
# earliest moment the hardware could perform it, so a buffer that is still being read when its refill is issued shows
# up as wrong results.  An mbarrier is emulated as a count of completed phases plus, in the word behind it, the transaction
# bytes announced by expect_tx and not yet delivered: a phase completes only when every announced byte has been copied
# (emu::tx_complete_check), and every bulk copy obeys cp.async.bulk's 16-byte alignment and size rule
# (emu::bulk_copy_check) - the two ways a wrong byte count or frame offset would hang or corrupt the GPU's copy.  A thread
# waiting for a phase that is not complete yet yields to the other threads of the block (the issuing thread may not have
# run yet), and a block in which everybody only waits is reported as a dead-lock.
PTX_STANDINS = {
    "mbar_init": "{ (void)count; reinterpret_cast<unsigned long long *>(bar)[0] = 0ull; reinterpret_cast<unsigned long long *>(bar)[1] = 0ull; }",
    "mbar_expect_tx": "{ reinterpret_cast<unsigned long long *>(bar)[1] += bytes; }",
    "bulk_g2s": "{ emu::bulk_copy_check(dst, src, bytes); memcpy(dst, src, bytes); unsigned long long *b = reinterpret_cast<unsigned long long *>(bar); "
                "b[1] -= bytes; emu::tx_complete_check(b); b[0] += 1ull; }",
    "bulk_g2s_multi": "{ emu::bulk_copy_check(dst, src, bytes); memcpy(dst, src, bytes); reinterpret_cast<unsigned long long *>(bar)[1] -= bytes; }",
    "mbar_host_commit": "{ unsigned long long *b = reinterpret_cast<unsigned long long *>(bar); emu::tx_complete_check(b); b[0] += 1ull; }",
    "mbar_wait": "{ while (((*reinterpret_cast<volatile unsigned long long *>(bar)) & 1ull) == parity) emu::spin_yield(); }",
    "fence_proxy_async": "{ }",
    "cp_async8": "{ if (valid) memcpy(smem_dst, gsrc, 8); else memset(smem_dst, 0, 8); }",
    "cp_async_commit": "{ }",
    "cp_async_wait": "{ }",
    "count_if_ge": "{ acc += (v >= lim) ? 1 : 0; }",
    "table_entry": "{ const double2 *t = tab_lane + (size_t)idx * TAB_REP; c01 = t[0]; c2f = t[(ICNV_EMIS_N + 1) * TAB_REP]; }",
}
DYN_SMEM = re.compile(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?(?P<type>[\w ]+?)\s+(?P<name>\w+)\[\];")

LAUNCH = re.compile(r"(?P<name>[A-Za-z_]\w*(?:<[^<>();]*>)?)\s*<<<(?P<cfg>.*?)>>>\s*\((?P<args>.*?)\);", re.S)


def replace_body(text: str, fn: str, body: str) -> str:
    """Swap the brace-delimited body of the device function `fn` (the definition, not its calls)."""
    m = re.search(r"(?:void|unsigned|long)\s+" + fn + r"\s*\([^)]*\)\s*\{", text)
    if not m:
        return text
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return text[:m.end() - 1] + body + text[i:]


def transform(text: str) -> tuple[str, int]:
    for fn, body in PTX_STANDINS.items():
        text = replace_body(text, fn, body)
    assert "asm volatile" not in text and "asm(" not in text, "inline PTX without a stand-in"
    text = DYN_SMEM.sub(lambda m: f"{m['type']} *{m['name']} = reinterpret_cast<{m['type']} *>(emu::dyn_smem);", text)
    return LAUNCH.subn(lambda m: f"EMU_LAUNCH({m['name']}, ({m['cfg']}), ({m['args']}));", text)


def build(force: bool = False) -> str:
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "emu", f) for f in os.listdir(os.path.join(HERE, "emu"))]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(s) <= os.path.getmtime(OUT) for s in srcs + [__file__]):
        return OUT
    gen = os.path.join(OUT_DIR, "src")
    shutil.rmtree(gen, ignore_errors=True)
    os.makedirs(gen)
    files = []
    for f in EMULATED:
        text, n = transform(open(os.path.join(CSRC, f)).read())
        assert "<<<" not in text, f"{f}: a launch was not recognised"
        dst = os.path.join(gen, f.replace(".cu", ".emu.cpp"))
        open(dst, "w").write(f"// generated from infercnv_b200/csrc/{f} by tests/host/build_emu.py ({n} launches rewritten)\n" + text)
        files.append(dst)
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    cmd = [gxx, "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-D__CUDACC__", "-DICNV_EMU", "-Wall", "-Wno-unknown-pragmas",
           "-Wno-attributes", "-Wno-unused-function", "-Wno-unused-variable", "-Wno-unused-but-set-variable", "-mfma",
           "-ffp-contract=off", "-pthread", "-rdynamic", "-fno-omit-frame-pointer", "-I", os.path.join(HERE, "emu"), "-I", CSRC, "-o", OUT, *files]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
