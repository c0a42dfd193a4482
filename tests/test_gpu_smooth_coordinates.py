"""K16 on the GPU: coordinate-weighted smoothing (icnv_smooth_coordinates_f64 / icnv_dev_smooth_coordinates_f64) within the
bound of include/infercnv_b200.h against the R-arithmetic restatement of tests/coordinates_reference.py, through api,
Engine and mirror.ops.  Under the host emulation (tests/test_smooth_coords_emulated_and_r.py) the full-size case and the
Engine are skipped."""
import os

import numpy as np
import pytest

from infercnv_b200 import _lib, api
from infercnv_b200._lib import InfercnvB200Error
from tests import coordinates_reference as cr
from tests.test_coordinates_reference import CASES, fixture, layout

pytestmark = pytest.mark.gpu
EMULATED = "_emu" in os.path.basename(_lib.LIB_PATH)
gpu_only = pytest.mark.skipif(EMULATED, reason="GPU only: too large for the host emulation")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", autouse=True)
def _init():
    api.init(0)


def values(G, C, seed):
    rng = np.random.default_rng(seed)
    return np.asfortranarray(rng.normal(size=(G, C)) * rng.choice([1.0, 1e3, 1e-3], size=C) + rng.normal(size=C))


@pytest.mark.parametrize("case", CASES)
def test_hand_built_layouts_within_the_bound(case):
    st, sp, cs, cl, W = layout(case)
    X = values(len(st), 37, len(case))          # two cell tiles, the second one partial
    Y = api.smooth_coordinates(X, cs, cl, st, sp, W)
    cr.check_coordinates(Y, X, cs, cl, st, sp, W)
    for s0, n in zip(cs, cl):
        if n < 2 or W < 2:
            assert np.array_equal(Y[s0:s0 + n], X[s0:s0 + n])


@pytest.mark.parametrize("W", [1e7, 1e6, 1e5, 2e4])
def test_example_coordinates_within_the_bound(W):
    X, st, sp, cs, cl = fixture()
    Y = api.smooth_coordinates(X, cs, cl, st, sp, W)
    share = cr.check_coordinates(Y, X, cs, cl, st, sp, W)
    print(f"W = {W:g}: {share:.5f} of the outputs bit-identical to R's arithmetic")


def gapped_layout(G):
    """Ranges with one-gene ranges and gaps (genes outside every range), as test_gpu_random_trees.layout."""
    if G < 4:
        return [0], [G]
    starts, lens, pos = [], [], 1   # gene 0 in no range
    for L in [1, 2, 40, 101, 102, 997]:
        if pos + L > G:
            break
        starts.append(pos)
        lens.append(L)
        pos += L + 1
    if pos < G - 1:
        starts.append(pos)
        lens.append(G - 1 - pos)
    return starts, lens


@pytest.mark.parametrize("G", [1, 2, 100, 300])
def test_ranges_with_gaps(G):
    rng = np.random.default_rng(G)
    st = np.floor(np.sort(rng.uniform(0, 3e6, G)))
    sp = st + rng.choice([500.0, 5e3, 4e4, 3e5], size=G)        # some genes long enough to leave holes
    X = values(G, 33, G + 1)
    cs, cl = gapped_layout(G)
    Y = api.smooth_coordinates(X, cs, cl, st, sp, 1e5)
    cr.check_coordinates(Y, X, cs, cl, st, sp, 1e5)
    inside = np.zeros(G, bool)
    for s, L in zip(cs, cl):
        inside[s:s + L] = True
        one = api.smooth_coordinates(X[s:s + L], [0], [L], st[s:s + L], sp[s:s + L], 1e5)
        assert np.array_equal(one, Y[s:s + L])                       # per range == whole call, bit for bit
    assert np.array_equal(Y[~inside], X[~inside])


def test_band_wider_than_a_chunk():
    """W spans the whole chromosome: 300-gene bands go through shared memory in several chunks."""
    G = 300
    st = np.arange(G) * 1000.0
    sp = st + 400.0
    X = values(G, 40, 9)
    Y = api.smooth_coordinates(X, [0], [G], st, sp, 1e9)
    cr.check_coordinates(Y, X, [0], [G], st, sp, 1e9)


def test_errors():
    st, sp = np.arange(10.0) * 10, np.arange(10.0) * 10 + 5
    X = np.ones((10, 3))
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth_coordinates(X, [0, 4], [5, 3], st, sp, 50.0)           # overlapping ranges
    assert e.value.code == -3
    bad = st.copy()
    bad[2] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth_coordinates(X, [0], [10], bad, sp, 50.0)
    assert e.value.code == -3
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth_coordinates(X, [0], [10], st, sp, float("nan"))
    assert e.value.code == -3
    X[3, 1] = np.nan
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth_coordinates(X, [0], [10], st, sp, 50.0)
    assert e.value.code == -5
    X[3, 1] = np.inf
    with pytest.raises(InfercnvB200Error) as e:
        api.smooth_coordinates(X, [0, 5], [1, 5], st, sp, 50.0)          # in a copied gene too
    assert e.value.code == -5


def test_mirror_op_and_its_hidden_spike():
    from mirror import ops
    st, sp, cs, cl, W = layout("hole_non_multiple")
    X = values(len(st), 6, 3)
    spike = ops.Infercnv(expr_data=values(len(st), 2, 4), gene_order_chr=np.zeros(len(st), int), gene_order_start=st,
                         gene_order_stop=sp)
    obj = ops.Infercnv(expr_data=X, gene_order_chr=np.zeros(len(st), int), gene_order_start=st, gene_order_stop=sp,
                       hspike=spike)
    out = ops.smooth_by_chromosome_coordinates(obj, W)
    assert np.array_equal(out.expr_data, api.smooth_coordinates(X, cs, cl, st, sp, W))
    assert np.array_equal(out.hspike.expr_data, api.smooth_coordinates(spike.expr_data, cs, cl, st, sp, 51))
    assert np.array_equal(obj.expr_data, X)                              # the input object is left alone


@gpu_only
def test_engine_equals_api():
    import torch
    from infercnv_b200.device import Engine
    st, sp, cs, cl = cr.synthetic_coordinates(2000, 1, GOLDEN)
    X = values(2000, 300, 5)
    want = api.smooth_coordinates(X, cs, cl, st, sp, 1e7)
    eng = Engine(0)
    T = torch.as_tensor(np.ascontiguousarray(X.T), device=eng.tdev)
    got = eng.smooth_coordinates(T, cs, cl, st, sp, 1e7).cpu().numpy().T
    assert np.array_equal(got, want)


@gpu_only
def test_full_size_10000_genes_20000_cells():
    import torch
    from infercnv_b200.device import Engine
    G, C = 10000, 20000
    st, sp, cs, cl = cr.synthetic_coordinates(G, 2, GOLDEN)
    eng = Engine(0)
    T = torch.log2(eng.synth(G, cs, cl, np.arange(C), C, 3) + 1.0)
    T = T - T.mean(dim=0, keepdim=True)
    Y = eng.smooth_coordinates(T, cs, cl, st, sp, 1e7)
    torch.cuda.synchronize()
    sample = np.sort(np.random.default_rng(4).choice(C, 24, replace=False))
    idx = torch.as_tensor(sample, device=eng.tdev)
    Xs = np.asfortranarray(T[idx].cpu().numpy().T)
    Ys = Y[idx].cpu().numpy().T
    share = cr.check_coordinates(Ys, Xs, cs, cl, st, sp, 1e7)
    print(f"full size: {share:.5f} of the sampled outputs bit-identical to R's arithmetic")
