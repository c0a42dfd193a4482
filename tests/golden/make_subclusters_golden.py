#!/usr/bin/env python
"""Extract the subcluster index lists stored in the reference's example object into tests/golden/example_subclusters.npz.

Run in the build container only (needs the read-only reference checkout); it writes that one file and nothing else:

    python tests/golden/make_subclusters_golden.py [/root/reference]

`data/infercnv_object_example.rda` keeps `@tumor_subclusters$subclusters`: per group ("tumor", "normal") a named list of
1-based cell indices ("tumor_s1", "normal_s1"), as define_signif_tumor_subclusters left them.  The file holds, per group
`<group>`, the subcluster names (`<group>_names`), their lists back to back (`<group>_idx`, 1-based, as in R) and the
offsets of each list (`<group>_off`).  This is the reference's data, reduced to arrays; nothing here is reference source
code.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rda_reader import named_list, read_rda  # noqa: E402


def main(ref: str) -> None:
    o = read_rda(os.path.join(ref, "data/infercnv_object_example.rda"))["infercnv_object_example"]
    sub = named_list(named_list(o.attr["tumor_subclusters"])["subclusters"])
    out = {}
    for grp, lst in sub.items():
        subs = named_list(lst)
        out[f"{grp}_names"] = np.array(list(subs))
        out[f"{grp}_idx"] = np.concatenate([np.asarray(v.value, dtype=np.int32) for v in subs.values()])
        out[f"{grp}_off"] = np.cumsum([0] + [len(v.value) for v in subs.values()]).astype(np.int32)
    np.savez_compressed(os.path.join(HERE, "example_subclusters.npz"), **out)
    print("example_subclusters.npz", {k: v.tolist() for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
