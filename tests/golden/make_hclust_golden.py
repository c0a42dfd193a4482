#!/usr/bin/env python
"""Extract the two hclust trees stored in the reference's example object into tests/golden/example_hclust.npz.

Run in the build container only (needs the read-only reference checkout); it writes that one file and nothing else:

    python tests/golden/make_hclust_golden.py [/root/reference]

`data/infercnv_object_example.rda` keeps `@tumor_subclusters$hc$tumor` and `$hc$normal`: ward.D2 linkages of the 10
observation and the 10 reference cells.  For each tree the file holds `merge` ((n - 1) x 2, R's convention), `height`,
`order` (1-based), the labels, and `cols` - the 0-based column of each label in `count.data` / `expr.data`.  This is the
reference's data, reduced to arrays; nothing here is reference source code.
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
    cell_names = list(o.attr["expr.data"].attr["dimnames"].value[1].value)
    hc = named_list(named_list(o.attr["tumor_subclusters"])["hc"])
    out = {}
    for name in ("tumor", "normal"):
        f = named_list(hc[name])
        n = len(f["order"].value)
        merge = np.asarray(f["merge"].value, dtype=np.int32).reshape((n - 1, 2), order="F")
        labels = [str(s) for s in f["labels"].value]
        assert str(f["method"].value[0]) == "ward.D2" and str(f["dist.method"].value[0]) == "euclidean"
        out[f"{name}_merge"] = merge
        out[f"{name}_height"] = np.asarray(f["height"].value, dtype=np.float64)
        out[f"{name}_order"] = np.asarray(f["order"].value, dtype=np.int32)
        out[f"{name}_labels"] = np.array(labels)
        out[f"{name}_cols"] = np.array([cell_names.index(s) for s in labels], dtype=np.int32)
    np.savez_compressed(os.path.join(HERE, "example_hclust.npz"), **out)
    print("example_hclust.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
