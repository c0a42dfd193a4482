"""infercnv_b200 - H100 (sm_90a) engine for inferCNV's smoothing + HMM hot path.

The product is `libinfercnv_b200.so` (C ABI in include/infercnv_b200.h, CUDA in csrc/).
The Python around it is plumbing:

* `infercnv_b200.api`      NumPy wrappers of the host-pointer ABI (what the R shim binds)
* `infercnv_b200.hmm`      the reference's HMM parameter tables (.get_HMM, .i3HMM_get_HMM)
* `infercnv_b200.device`   torch-tensor wrappers of the device-pointer ABI, sharding over GPUs (one process per GPU)
* `infercnv_b200.dist`     the shard planner
* `infercnv_b200/r/`       the R shim and the drop-in closures (the reference-facing boundary)

(`mirror/ops.py` at the repository root - the reference's R function names on top of `api`, for tests and examples - is
not part of the product.)
"""
from . import _lib  # noqa: F401

__version__ = "0.1.0"
