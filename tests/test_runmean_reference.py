"""CPU pins of tests/runmean_reference.py: the long-double window rule against a literal transcription of caTools' running
sum, and the NumPy generator against the oracle's C twin, with the permutations it defines checked for shape and
uniformity."""
import ctypes
import os
import re
import shutil
import subprocess
from math import factorial
from itertools import permutations as all_orders

import numpy as np
import pytest
from scipy.stats import chisquare

from tests import runmean_reference as rr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n,k", [(7, 12), (8, 12), (6, 6), (9, 1), (2, 3), (2, 2), (5, 3), (40, 101), (40, 101 - 60),
                                 (50, 11), (50, 10), (13, 4)])
def test_restatement_matches_the_catools_transcription(n, k):
    x = np.random.default_rng(n * 100 + k).normal(size=n) * 10.0 ** np.random.default_rng(k).integers(-3, 4, size=n)
    ref, tol = rr.runmean_ld(x, k)
    want = np.array(rr.catools_transcription(x, k))
    # the transcription is exact up to its final rounding to double
    assert np.all(np.abs(ref[:, 0].astype(np.float64) - want) <= tol[:, 0] + 2 * rr.U * np.abs(want)), (ref[:, 0], want)


def test_five_gene_hand_case():
    x = [1.0, 2.0, 4.0, 8.0, 16.0]
    # k = 3: windows [0,1] [0,2] [1,3] [2,4] [3,4]
    assert rr.catools_transcription(x, 3) == [1.5, 7 / 3, 14 / 3, 28 / 3, 12.0]
    ref, _ = rr.runmean_ld(x, 3)
    assert np.allclose(ref[:, 0].astype(np.float64), [1.5, 7 / 3, 14 / 3, 28 / 3, 12.0], rtol=0, atol=1e-15)
    # k = 4 (even): k2 = 2, k1 = 1 - windows [0,2] [0,3] [1,4] [2,4] [3,4]
    assert rr.catools_transcription(x, 4) == [7 / 3, 15 / 4, 30 / 4, 28 / 3, 12.0]


def test_window_rule_edges():
    assert [rr.window(p, 4, 10) for p in range(4)] == [(0, 2), (0, 3), (1, 3), (2, 3)]   # k > n, n even: k1 = k2 - 1
    assert [rr.window(p, 5, 10) for p in range(5)] == [(0, 2), (0, 3), (0, 4), (1, 4), (2, 4)]
    assert [rr.window(p, 2, 3) for p in range(2)] == [(0, 1), (1, 1)]   # k' = 2: k2 = 1, k1 = 0
    assert [rr.window(p, 3, 1) for p in range(3)] == [(0, 0), (1, 1), (2, 2)]


def test_copies_and_ranges():
    x = np.arange(10.0)[:, None] ** 2
    ref, tol = rr.runmean_ld(x, 1)
    assert np.array_equal(ref.astype(np.float64), x) and not tol.any()
    ref, _ = rr.runmean_ld(x, 3, [0, 4, 5], [3, 1, 5])   # gene 3 outside every range, range [4, 5) has one gene
    assert ref[3, 0] == 9.0 and ref[4, 0] == 16.0
    assert np.isclose(float(ref[0, 0]), 0.5) and np.isclose(float(ref[9, 0]), (64 + 81) / 2)


def test_bound_is_tight_enough_to_mean_something():
    x = np.random.default_rng(3).normal(size=(2000, 2))
    ref, tol = rr.runmean_ld(x, 101)
    assert np.median(tol / np.abs(ref.astype(np.float64))) < 3 * rr.U   # a few ulp of the mean, not a drift allowance


@pytest.fixture(scope="module")
def oracle_hash3(tmp_path_factory):
    """The oracle's syn_hash3 (and the syn_mix64 it calls), cut out of oracle/infercnv_oracle.c and compiled alone."""
    src = open(os.path.join(ROOT, "oracle", "infercnv_oracle.c")).read()
    parts = []
    for name in ("syn_mix64", "syn_hash3"):
        m = re.search(r"static uint64_t " + name + r"\(.*?\n}\n", src, re.S)
        assert m, name
        parts.append(m.group(0).replace("static ", "", 1))
    d = tmp_path_factory.mktemp("hash3")
    c = d / "h.c"
    c.write_text("#include <stdint.h>\n" + "\n".join(parts))
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    so = d / "h.so"
    subprocess.check_call([gcc, "-O1", "-shared", "-fPIC", "-o", str(so), str(c)])
    lib = ctypes.CDLL(str(so))
    lib.syn_hash3.restype = ctypes.c_uint64
    lib.syn_hash3.argtypes = [ctypes.c_uint64] * 4
    return lib.syn_hash3


def test_numpy_generator_equals_the_oracle_twin(oracle_hash3):
    rng = np.random.default_rng(1)
    for _ in range(200):
        s, a, b, c = (int(v) for v in rng.integers(0, 2 ** 63, size=4, dtype=np.int64))
        assert int(rr.hash3(s, a, b, c)) == oracle_hash3(s, a, b, c)
    for s, a, b, c in [(0, 0, 0, 0), (2 ** 64 - 1, 99, 9999, 65535), (12345, 0, 3, 1)]:
        assert int(rr.hash3(s, a, b, c)) == oracle_hash3(s, a, b, c)


def test_every_slice_is_a_permutation():
    for n in (2, 3, 33, 257):
        for p in (0, 1, 99):
            pi = rr.permutations(7, p, 50, n)
            assert np.array_equal(np.sort(pi, axis=1), np.broadcast_to(np.arange(n), (50, n)))


def test_raw_hash3_orders_are_not_uniform_but_keys_are():
    """Why the key is mix64(hash3(...)): ordering by hash3 alone reaches only 8 of the 24 orders of four positions."""
    g = np.arange(500, dtype=np.uint64)[:, None]
    i = np.arange(4, dtype=np.uint64)[None, :]
    raw = {tuple(r) for r in np.argsort(rr.hash3(5, np.uint64(0), g, i), axis=1, kind="stable")}
    assert len(raw) == 8
    assert len({tuple(r) for r in rr.permutations(5, 0, 500, 4)}) == 24


def test_orders_of_four_are_uniform():
    # n = 4: all 24 orders at the expected frequency over (p, g) slices, chi-square at a fixed seed
    pi = np.concatenate([rr.permutations(2024, p, 2000, 4) for p in range(12)])
    code = {o: i for i, o in enumerate(all_orders(range(4)))}
    counts = np.bincount([code[tuple(r)] for r in pi], minlength=factorial(4))
    assert counts.sum() == 24000
    assert chisquare(counts).pvalue > 1e-3, counts
