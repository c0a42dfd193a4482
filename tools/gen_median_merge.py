#!/usr/bin/env python
"""Generates infercnv_b200/csrc/icnv_median_merge.inc: the comparator networks of the shared-merge median filter
(apply_median_filtering, window_size 7 = 9 x 9 taps; K4 in DESIGN.md) on 32-bit keys.

A 9 x 9 window is 9 sorted runs of 9 keys (one run per list position, the 9 genes around the output).  Outputs that are
neighbours along the cell list share 8 of their 9 runs, and the merges are arranged so that the shared part is built once:

  sort9     25 comparators (optimal), one run per halo position
  merge9    run + run               -> P (18 keys, pairs of consecutive list positions)
  merge18   P + P                   -> Q (36 keys, four consecutive positions)
  core      Q + Q, only ranks 30..43 of the 72 keys (the 14 that can still be ranks 39..43 of a window once any 9 more keys join)
  select    those 14 + the one run a window adds -> ranks 39..43 of the 81 keys

Merges are Batcher odd-even merges on power-of-two padded lists with the padding folded away symbolically; `core` and
`select` are the full merges with every comparator that no requested output depends on removed (and half-comparators where
only the min or the max is needed).  Every network is checked here with the 0-1 principle before it is written.

    python tools/gen_median_merge.py [--check-only]
"""
import itertools
import os
import sys

INF = "INF"


class Net:
    def __init__(self):
        self.ops = []   # (kind, out, a, b) in SSA form
        self.n = 0

    def new(self):
        self.n += 1
        return self.n - 1

    def mn(self, a, b):
        if a == INF:
            return b
        if b == INF:
            return a
        o = self.new()
        self.ops.append(("min", o, a, b))
        return o

    def mx(self, a, b):
        if a == INF or b == INF:
            return INF
        o = self.new()
        self.ops.append(("max", o, a, b))
        return o

    def cs(self, a, b):
        return self.mn(a, b), self.mx(a, b)


def merge_pow2(net, A, B):
    n = len(A)
    assert n == len(B) and (n & (n - 1)) == 0
    if n == 1:
        return list(net.cs(A[0], B[0]))
    V = merge_pow2(net, A[0::2], B[0::2])
    W = merge_pow2(net, A[1::2], B[1::2])
    out = [V[0]]
    for i in range(len(W) - 1):
        out += list(net.cs(W[i], V[i + 1]))
    out.append(W[-1])
    return out


def merge(net, A, B):
    p = 1
    while p < max(len(A), len(B)):
        p *= 2
    out = merge_pow2(net, A + [INF] * (p - len(A)), B + [INF] * (p - len(B)))
    res = out[:len(A) + len(B)]
    assert all(x != INF for x in res) and all(x == INF for x in out[len(A) + len(B):])
    return res


def dce(ops, needed):
    need, keep = set(needed), []
    for op in reversed(ops):
        if op[1] in need:
            keep.append(op)
            need.update(op[2:4])
    keep.reverse()
    return keep


def evaluate(ops, env):
    for k, o, a, b in ops:
        env[o] = min(env[a], env[b]) if k == "min" else max(env[a], env[b])
    return env


SORT9 = [[(0, 3), (1, 7), (2, 5), (4, 8)], [(0, 7), (2, 4), (3, 8), (5, 6)], [(0, 2), (1, 3), (4, 5), (7, 8)],
         [(1, 4), (3, 6), (5, 7)], [(0, 1), (2, 4), (3, 5), (6, 8)], [(2, 3), (4, 5), (6, 7)], [(1, 2), (3, 4), (5, 6)]]


def build_sort9():
    net = Net()
    ins = [net.new() for _ in range(9)]
    w = list(ins)
    for layer in SORT9:
        for i, j in layer:
            w[i], w[j] = net.cs(w[i], w[j])
    for bits in itertools.product((0, 1), repeat=9):   # 0-1 principle
        env = evaluate(net.ops, dict(zip(ins, bits)))
        r = [env[x] for x in w]
        assert r == sorted(r), "sort9 network is not a sorting network"
    return net.ops, [ins], w


def build_merge(m, n, lo=None, hi=None):
    """merge of sorted lists of m and n keys; outputs ranks lo..hi (1-based, inclusive; default all)."""
    net = Net()
    A = [net.new() for _ in range(m)]
    B = [net.new() for _ in range(n)]
    out = merge(net, A, B)
    outs = out if lo is None else out[lo - 1:hi]
    ops = dce(net.ops, outs)
    first = 0 if lo is None else lo - 1
    for i in range(m + 1):          # 0-1 principle on sorted inputs
        for j in range(n + 1):
            env = evaluate(ops, dict(zip(A + B, [0] * (m - i) + [1] * i + [0] * (n - j) + [1] * j)))
            want = sorted([0] * (m - i) + [1] * i + [0] * (n - j) + [1] * j)[first:first + len(outs)]
            assert [env[o] for o in outs] == want, (m, n, lo, hi, i, j)
    return ops, [A, B], outs


def emit(name, ops, ins, outs, in_names, out_name, doc):
    rename = {}
    for arr, nm in zip(ins, in_names):
        for i, v in enumerate(arr):
            rename[v] = f"{nm}[{i}]"
    lines = [f"// {doc}: {len(ops)} min / max operations", f"#define {name}({', '.join(in_names + [out_name])}) do {{ \\"]
    for k, o, a, b in ops:
        rename[o] = f"t{o}_"
        lines.append(f"    const unsigned t{o}_ = mf_{k}({rename[a]}, {rename[b]}); \\")
    for i, o in enumerate(outs):
        lines.append(f"    {out_name}[{i}] = {rename[o]}; \\")
    lines.append("} while (0)")
    return "\n".join(lines)


def main():
    parts = ["// icnv_median_merge.inc - generated by tools/gen_median_merge.py; do not edit.  See that file for what the networks are.",
             "// mf_min / mf_max are defined by the includer (unsigned min / max: VIMNMX.U32 on sm_90a)."]
    ops, ins, outs = build_sort9()
    # sort9 works in place on one array: emit as input k, output k
    parts.append(emit("MF_SORT9", ops, ins, outs, ["k_"], "r_", "sort 9 keys (25 comparators, 7 layers)"))
    counts = {"sort9": len(ops)}
    for name, m, n, lo, hi, doc in (("MF_MERGE9", 9, 9, None, None, "two sorted runs of 9 -> 18 sorted keys"),
                                    ("MF_MERGE18", 18, 18, None, None, "two sorted lists of 18 -> 36 sorted keys"),
                                    ("MF_CORE", 36, 36, 30, 43, "two sorted lists of 36 -> ranks 30..43 of the 72 keys (14 sorted keys)"),
                                    ("MF_SELECT", 14, 9, 10, 14, "14 core keys + a sorted run of 9 -> ranks 10..14 of the 23, i.e. ranks 39..43 of the window's 81 keys")):
        ops, ins, outs = build_merge(m, n, lo, hi)
        parts.append(emit(name, ops, ins, outs, ["a_", "b_"], "o_", doc))
        counts[name] = len(ops)
    text = "\n\n".join(parts) + "\n"
    print("operations:", counts, file=sys.stderr)
    if "--check-only" in sys.argv:
        return
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "infercnv_b200", "csrc", "icnv_median_merge.inc")
    open(out, "w").write(text)
    print(out)


if __name__ == "__main__":
    main()
