"""Non-DE masking across ranks (Engine.mask_non_de_sharded, tools/check_de_sharded.py): with the genes split over 2, 3 and 4
ranks, p_raw, p_adj and each rank's columns of Y equal api.mask_non_de_genes on the gathered matrix byte for byte, for
reference groups cut across ranks, whole subclusters, a rank without listed cells, tie-laden data, both Wilcoxon regimes, the
t test and the three rules, and a NaN on one rank raises ICNV_E_NONFINITE on every rank.  On a one-GPU box the ranks share
cuda:0 and the exchange goes through gloo / host memory; with >= world GPUs the same script runs over NCCL.  The host entry
point over several device slots (icnv_init_devices) is checked against one slot when the box has two GPUs."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_mask_is_bitwise_equal_to_one_call(world):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, ICNV_DIST_BACKEND="gloo", ICNV_ONE_GPU="1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "check_de_sharded.py")],
                       capture_output=True, text=True, timeout=900, env=env)
    tail = r.stdout[-2500:] + r.stderr[-2500:]
    assert r.returncode == 0 and "BITWISE EQUAL" in r.stdout, tail


@pytest.mark.gpu
def test_host_entry_over_device_slots_equals_one_slot():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: icnv_init_devices does not take a device twice")
    sys.path.insert(0, ROOT)
    from infercnv_b200 import api
    from tests import de_shards
    X, _, refs, subs = de_shards.make_case(1, 2000, [300, 200], [100, 40, 400, 3], seed=9)
    api.init(0)
    one = api.mask_non_de_genes(X, refs, subs, seed=4)
    try:
        api.init_devices(None)
        many = api.mask_non_de_genes(X, refs, subs, seed=4)
    finally:
        api.init(0)
    for a, b in zip(one, many):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
