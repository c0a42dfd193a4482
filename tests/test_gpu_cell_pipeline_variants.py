"""Every instantiation of the fused cell pipeline (icnv_dev_cell_pipeline_f64: 7 of the two-buffer cell_pipeline3_kernel, 7 of
the single-buffer cell_pipeline4_kernel) against the extended-precision reference of tests/cellpipe_reference.py.

The tuning switches ICNV_CELL_KERNEL / _NT / _PADQ / _LFIX (read at icnv_init, hence api.reinit()) walk the variants; which
instantiation actually ran is read back with icnv_debug_cell_kernel, so a change of the selection rule cannot silently drop a
variant from the sweep.  For every case:
  (a) every variant is within the per-element error bound of its prefix-sum formulation (tests/cellpipe_reference.py);
  (b) variants that share a slice partition are bit-identical.  The bits are fixed by the segment table (slice length L on
      the layout) - the summation order of the prefix sums P and Q - not by the kernel family, the padded-Q layout or the
      unrolled loops; mean centring adds the order of its reduction, which in the single-buffer kernel also depends on the
      thread count;
  (c) the default selection agrees with the reference as closely as the parity tests require of it against the oracle.
The gene counts sit on both sides of each selection boundary (thread count, two-buffer fit, padded-Q fit, the single-buffer
kernel's limit), the layouts exercise the per-chromosome bulk copies of the single-buffer kernel (odd starts / ends, tiny
and empty chromosomes), odd G and a column stride G + 1 the element-wise load path, and the cell counts the persistent loop.

Runs on an H100 (-m gpu) and, for G <= EMU_MAX_GENES, under the host emulation (tests/host/run_emulated.py), where device
buffers are host memory.  `pytest -s` prints the coverage table: instantiation, cases, worst error as a fraction of the bound.
"""
import ctypes as ct
import os

import numpy as np
import pytest

from infercnv_b200 import _lib
from oracle import oracle as orc
from tests import cellpipe_reference as cref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not cref.HAS_EXTENDED, reason="np.longdouble is not an extended type here")]

EMULATED = os.path.basename(_lib.LIB_PATH) != "libinfercnv_b200.so"
EMU_MAX_GENES = 6200       # the host emulation runs the cases up to this size (and the 6144 / 6145 boundary)
EMU_SM_COUNT = 4           # what tests/host/emu/cuda_runtime.h reports

CONFIGS = [
    {},
    {"ICNV_CELL_PADQ": "0"},
    {"ICNV_CELL_LFIX": "0"},
    {"ICNV_CELL_NT": "256"}, {"ICNV_CELL_NT": "512"}, {"ICNV_CELL_NT": "1024"},
    {"ICNV_CELL_NT": "256", "ICNV_CELL_PADQ": "0"}, {"ICNV_CELL_NT": "512", "ICNV_CELL_PADQ": "0"},
    {"ICNV_CELL_NT": "1024", "ICNV_CELL_PADQ": "0"},
    {"ICNV_CELL_KERNEL": "4"}, {"ICNV_CELL_KERNEL": "4", "ICNV_CELL_LFIX": "0"},
    {"ICNV_CELL_KERNEL": "4", "ICNV_CELL_NT": "256"}, {"ICNV_CELL_KERNEL": "4", "ICNV_CELL_NT": "512"},
    {"ICNV_CELL_KERNEL": "4", "ICNV_CELL_NT": "1024"}, {"ICNV_CELL_KERNEL": "4", "ICNV_CELL_NT": "1024", "ICNV_CELL_LFIX": "0"},
    {"ICNV_CELL_KERNEL": "4", "ICNV_CELL_NT": "512", "ICNV_CELL_LFIX": "0"},
]
if EMULATED:   # the unrolled slices (L = 11 / 21) need 10 000 genes or more: no instantiation to reach at the emulated sizes
    CONFIGS = [c for c in CONFIGS if "ICNV_CELL_LFIX" not in c]
SWITCHES = ("ICNV_CELL_KERNEL", "ICNV_CELL_NT", "ICNV_CELL_PADQ", "ICNV_CELL_LFIX")

ALL_INSTANTIATIONS = {(3, nt, 1, pq, 0) for nt in (256, 512, 1024) for pq in (0, 1)} | {(3, 1024, 1, 1, 11)} | \
    {(4, 256, 4, 0, 0), (4, 256, 1, 0, 0), (4, 512, 2, 0, 21), (4, 512, 2, 0, 0), (4, 512, 1, 0, 0), (4, 1024, 1, 0, 21),
     (4, 1024, 1, 0, 0)}
NAMES = {3: "cell_pipeline3_kernel<{1}, {3}, {4}>", 4: "cell_pipeline4_kernel<{1}, {2}, 1024, {4}>"}

COVER = {}          # instantiation -> [cases, worst error / bound]
SPECIAL = {}        # "element-wise load" / "refused with -4" -> cases
DONE = set()        # tests of this module that ran to the end


def _name(sel):
    s = list(sel[:5])
    if s[0] == 3:
        s[3] = "true" if s[3] else "false"
    return NAMES[sel[0]].format(*s)


def _note(sel, ratio):
    e = COVER.setdefault(tuple(sel[:5]), [0, 0.0])
    e[0] += 1
    e[1] = max(e[1], ratio)


# ---- device buffers: torch CUDA tensors on the GPU, host memory under the emulation --------------------------------------
@pytest.fixture(scope="module")
def api():
    from infercnv_b200 import api as a
    a.init(0)
    return a


def _torch():
    import torch
    return torch


def _dev():
    return _torch().device("cpu") if EMULATED else _torch().device("cuda", 0)


def _stream():
    if EMULATED:
        return ct.c_void_p(1)
    from infercnv_b200 import device
    return device._stream_ptr()


def _sm_count():
    return EMU_SM_COUNT if EMULATED else _torch().cuda.get_device_properties(0).multi_processor_count


def _configure(api, monkeypatch, env):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    api.reinit()   # the switches are read once, at icnv_init


class Case:
    """One call of the device entry point: X (C, G) cells as rows, stage options, optional column list / strides."""

    def __init__(self, name, cs, cl, X, opts, cols=None, ldx=None, ldy=None, refuse=False):
        self.name, self.X, self.opts, self.refuse = name, np.ascontiguousarray(X, dtype=np.float64), dict(opts), refuse
        self.cs, self.cl = np.ascontiguousarray(cs, dtype=np.int32), np.ascontiguousarray(cl, dtype=np.int32)
        self.C, self.G = self.X.shape
        self.cols = None if cols is None else np.ascontiguousarray(cols, dtype=np.int32)
        self.ldx, self.ldy = ldx or self.G, ldy or self.G
        self._ref = {}
        self._dev = None

    @property
    def rows(self):
        return self.X if self.cols is None else self.X[self.cols]

    def element_wise_load(self):
        """True when some column's address or length breaks the 16-byte rule of the bulk copy"""
        return self.G % 2 == 1 or self.ldx % 2 == 1

    def upload(self):
        if self._dev is None:
            torch = _torch()
            buf = np.zeros((self.C, self.ldx))
            buf[:, :self.G] = self.X
            d = {"X": torch.from_numpy(buf).to(_dev())}
            for k in ("lo1", "hi1", "mid1", "lo2", "hi2", "mid2"):
                if self.opts.get(k) is not None:
                    d[k] = torch.from_numpy(np.ascontiguousarray(self.opts[k], dtype=np.float64)).to(_dev())
            if self.cols is not None:
                d["cols"] = torch.from_numpy(self.cols).to(_dev())
            self._dev = d
        return self._dev

    def run(self):
        """-> (rc, Y (n_cols, G) or None, err flag, selected instantiation)"""
        torch = _torch()
        d = self.upload()
        n = self.C if self.cols is None else len(self.cols)
        Y = torch.full((n, self.ldy), 12345.0, dtype=torch.float64, device=_dev())
        flag = torch.zeros(1, dtype=torch.int32, device=_dev())
        o = self.opts
        p = {k: (d[k].data_ptr() if k in d else None) for k in ("lo1", "hi1", "mid1", "lo2", "hi2", "mid2")}
        rc = _lib.load().icnv_dev_cell_pipeline_f64(
            d["X"].data_ptr(), self.G, self.ldx, d["cols"].data_ptr() if "cols" in d else None, n, Y.data_ptr(), self.ldy,
            self.cs.ctypes.data, self.cl.ctypes.data, len(self.cs), int(o.get("apply_log", False)), p["lo1"], p["hi1"], p["mid1"],
            float(o.get("threshold", 0.0)), int(o.get("window", 0)), int(o.get("center", 0)), p["lo2"], p["hi2"], p["mid2"],
            int(o.get("apply_exp2", False)), flag.data_ptr(), _stream())
        from infercnv_b200 import api
        sel = api.last_cell_kernel()
        if rc:
            return rc, None, 0, sel
        Yh = Y.cpu().numpy()
        assert np.all(Yh[:, self.G:] == 12345.0), f"{self.name}: write past G in an output column (ldy = {self.ldy})"
        return 0, Yh[:, :self.G].copy(), int(flag.cpu().item()), sel

    def reference(self, L, NW):
        key = (L, NW)
        if key not in self._ref:
            self._ref[key] = cref.cell_pipeline(self.rows, self.cs, self.cl, L=L, NW=NW, **self.opts)
        return self._ref[key]


def _partition_key(case, sel):
    # bits follow the segment table (slice length L on this layout); mean centring also follows its reduction order
    if case.opts.get("center", 0) == 2:
        return (sel[5], sel[0], sel[1] if sel[0] == 4 else 0)
    return (sel[5],)


def sweep(api, monkeypatch, cases, configs=None):
    """Run every case under every configuration, then check (a), (b), (c) for each case."""
    configs = CONFIGS if configs is None else configs
    res = [[] for _ in cases]
    try:
        for env in configs:
            _configure(api, monkeypatch, env)
            for i, c in enumerate(cases):
                res[i].append((env,) + c.run())
    finally:
        _configure(api, monkeypatch, {})
    for c, rr in zip(cases, res):
        _check(c, rr)
        c._dev = None


def _check(case, rr):
    if case.refuse:
        # the default selection refuses; a forced thread count may still fit (smaller reduction scratch): then it is checked
        for env, rc, Y, flag, sel in rr:
            if rc == -4 or not env:
                assert rc == -4 and sel == (0,) * 6, (case.name, env, rc, sel)
        SPECIAL["refused with -4"] = SPECIAL.get("refused with -4", 0) + 1
        rr = [t for t in rr if t[1] != -4]
    first = {}
    for env, rc, Y, flag, sel in rr:
        assert rc == 0, (case.name, env, rc, _lib.load().icnv_last_error())
        assert sel[0] in (3, 4) and sel[5] > 0, (case.name, env, sel)
        assert flag == 0, (case.name, env)
        want, bound = case.reference(sel[5], sel[1] // 32)
        r = cref.error_ratio(Y, want, bound)
        assert r <= 1.0, f"{case.name} {_name(sel)} (L = {sel[5]}, {env}): error {r:.3g} x the bound"
        _note(sel, r)
        if case.element_wise_load():
            k = f"element-wise load, cell_pipeline{sel[0]}_kernel"
            SPECIAL[k] = SPECIAL.get(k, 0) + 1
        key = _partition_key(case, sel)
        if key in first:
            sel0, Y0 = first[key]
            assert np.array_equal(Y.view(np.uint64), Y0.view(np.uint64)), \
                f"{case.name}: {_name(sel)} and {_name(sel0)} share slices of {sel[5]} genes but differ in " \
                f"{int(np.sum(Y != Y0))} values"
        else:
            first[key] = (sel, Y)
        if not env and case.opts.get("apply_exp2"):
            # (c) the default selection, as tightly as the parity tests hold the smooth block (2^x: no values near 0) to the oracle
            w = want.astype(np.float64)
            np.testing.assert_allclose(Y, w, rtol=1e-10, atol=1e-12 * max(1.0, float(np.max(np.abs(w)))), err_msg=case.name)


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _layout(lens):
    lens = np.asarray(lens, dtype=np.int32)
    return np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32), lens


def _bench_layout(G):
    import bench
    return bench.chr_layout(G)


def _data(rng, G, C, special=True):
    X = rng.gamma(2.0, 1.5, size=(C, G))
    X[rng.random((C, G)) < 0.3] = 0.0
    if special and C >= 4:
        X[1] = 2.5                                  # a constant column
        X[2, rng.random(G) < 0.5] = 1.75            # ties: far more than CAND_MAX values in the median's middle bin
        X[3, rng.choice(G, size=min(G, 7), replace=False)] = -1.0   # x + 1 == 0
    return X


def _opts(rng, X, kind="pass2", window=101, **over):
    """stage options; bounds drawn around the data (dead bands of the reference-mean step)"""
    G = X.shape[1]
    with np.errstate(divide="ignore"):
        base = np.log2(np.maximum(X, 0.0) + 1.0)
    lo = np.quantile(base, 0.4, axis=0) - 0.05
    hi = lo + rng.uniform(0.0, 0.3, size=G)
    lo2 = -rng.uniform(0.0, 0.2, size=G)
    hi2 = rng.uniform(0.0, 0.2, size=G)
    o = {
        "pass2": dict(apply_log=True, lo1=lo, hi1=hi, threshold=3.0, window=window, center=1, lo2=lo2, hi2=hi2, apply_exp2=True),
        "pass1": dict(apply_log=True, lo1=lo, hi1=hi, threshold=3.0, window=window, center=1),
        "mid": dict(apply_log=False, mid1=0.5 * (lo + hi), threshold=0.0, window=window, center=2, mid2=0.5 * (lo2 + hi2)),
        "stage_d": dict(lo2=lo2, hi2=hi2, apply_exp2=True),
        "stage_d_mid": dict(mid2=0.5 * (lo2 + hi2), apply_exp2=True),
    }[kind]
    o.update(over)
    return o


def _no_minus_one_under_log(X, o):
    if o.get("apply_log") and not o.get("threshold", 0.0) > 0.0:
        X = X.copy()
        X[X == -1.0] = 0.0     # log2(0) = -Inf is only finite after the clamp
    return X


def _fits(G):
    return G <= EMU_MAX_GENES or not EMULATED


# ---- tests -------------------------------------------------------------------------------------------------------------
def _probe(api, G):
    """default selection for G genes in the benchmark's layout (one cell): the instantiation, or None when refused"""
    cs, cl = _bench_layout(G)
    rng = np.random.default_rng(G)
    X = _data(rng, G, 1, special=False)
    rc, _, _, sel = Case("probe", cs, cl, X, _opts(rng, X)).run()
    assert rc in (0, -4), rc
    return None if rc else sel


def _last_true(pred, lo, hi):
    assert pred(lo) and not pred(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pred(mid) else (lo, mid)
    return lo


def test_selection_boundaries_by_gene_count(api, monkeypatch):
    """2048 / 2049 and 6144 / 6145 (256 -> 512 -> 1024 threads), the last G where the padded-Q layout fits and the first
    where it does not, the last G where the two-buffer kernel fits and the first where the single-buffer kernel takes over,
    the benchmark's 10 000 genes (slices of 11 / 21), 20 000 genes, and the last G the single-buffer kernel accepts next to
    the first it refuses with ICNV_E_UNSUPPORTED - all in the benchmark's 22-chromosome layout at window 101."""
    _configure(api, monkeypatch, {})
    Gs = [2048, 2049, 6144, 6145]
    expect = {2048: (3, 256), 2049: (3, 512), 6144: (3, 512), 6145: (3, 1024)}
    if not EMULATED:
        gq = _last_true(lambda G: (s := _probe(api, G)) is not None and s[0] == 3 and s[3] == 1, 10000, 20000)
        g3 = _last_true(lambda G: (s := _probe(api, G)) is not None and s[0] == 3, gq, 20000)
        g4 = _last_true(lambda G: _probe(api, G) is not None, 20000, 40000)
        assert gq < g3 or gq == g3
        print(f"\n[cell pipeline] padded-Q layout up to {gq} genes, two-buffer kernel up to {g3}, single-buffer up to {g4} "
              f"(window 101, 22 chromosomes)")
        Gs += sorted({gq, gq + 1, g3, g3 + 1, 10000, 20000, g4})
        expect.update({gq: (3, 1024, 1, 1), g3: (3,), g3 + 1: (4,), 10000: (3, 1024, 1, 1, 11, 11), 20000: (4, 1024, 1, 0, 21, 21),
                       g4: (4,)})
        if gq + 1 <= g3:
            expect[gq + 1] = (3, 1024, 1, 0)
    rng = np.random.default_rng(7)
    cases = []
    for G in Gs:
        cs, cl = _bench_layout(G)
        X = _data(rng, G, 4)
        cases.append(Case(f"G={G}", cs, cl, X, _opts(rng, X)))
    if not EMULATED:
        cs, cl = _bench_layout(g4 + 1)
        X = _data(rng, g4 + 1, 1, special=False)
        cases.append(Case(f"G={g4 + 1}", cs, cl, X, _opts(rng, X), refuse=True))
    sweep(api, monkeypatch, cases)
    for c in cases:
        if c.refuse:
            continue
        _, _, _, sel = c.run()
        want = expect.get(c.G)
        if want is not None:
            assert sel[:len(want)] == want, (c.G, sel, want)
    if not EMULATED:
        _configure(api, monkeypatch, {"ICNV_CELL_KERNEL": "4"})
        try:
            assert _probe(api, 10000) == (4, 512, 2, 0, 21, 21)   # the single-buffer kernel at the c3 size: two CTAs per SM
        finally:
            _configure(api, monkeypatch, {})
        # (c) through the host entry point, against the oracle, as the parity tests do
        for G in (6145, g3 + 1):
            cs, cl = _bench_layout(G)
            counts = rng.poisson(rng.lognormal(0.5, 1.0, size=(G, 1)) * rng.lognormal(0, 0.2, size=(1, 12))).astype(np.float64)
            refs = [np.arange(0, 3), np.arange(3, 5)]
            got = api.smooth_block(counts, cs, cl, refs)
            want = orc.smooth_block(counts, cs, cl, refs, nthreads=orc.max_threads())
            assert np.max(np.abs(got - want) / np.abs(want)) < 1e-10
    DONE.add("boundaries")


LAYOUTS = {
    # odd starts and odd ends everywhere, one- and two-gene chromosomes, chromosomes shorter than h = 50, and chromosomes of
    # 2h + 1 .. 2h + 1 + a slice (a slice can see both ends), an empty chromosome inside and one at the end
    "odd_ends": [301, 1, 2, 149, 77, 103, 105, 111, 0, 3, 49, 1200, 51, 99, 2, 1, 777, 0],
    # 30 chromosomes, even total
    "thirty": [120, 97, 88, 201, 13, 1, 64, 333, 2, 150, 101, 102, 47, 90, 500, 31, 17, 250, 3, 99, 180, 41, 60, 77, 111, 140,
               1, 200, 19, 93],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_chromosome_layouts(api, monkeypatch, layout):
    rng = np.random.default_rng(11)
    cs, cl = _layout(LAYOUTS[layout])
    G = int(cl.sum())
    X = _data(rng, G, 5)
    cases = [Case(f"{layout} w={w}", cs, cl, X, _opts(rng, X, window=w)) for w in (101, 3)]
    cases.append(Case(f"{layout} pass1", cs, cl, X, _opts(rng, X, "pass1")))
    sweep(api, monkeypatch, cases)
    DONE.add("layout_" + layout)


def test_stage_options(api, monkeypatch):
    """log on / off, dead band / mid subtraction, threshold 0, windows 0, 1, 3, 101 and one longer than every chromosome,
    centring none / median / mean, 2^x on / off, the stage-D-only call device.py makes for the leading reference columns;
    constant, tie-dominated and x = -1 columns (the median's fallback selection, log2(0))."""
    rng = np.random.default_rng(12)
    cs, cl = _layout([400, 1, 350, 77, 2, 612, 150, 290, 33, 501, 199, 285, 100])
    G = int(cl.sum())
    X0 = _data(rng, G, 5)
    longest = int(cl.max())
    variants = [
        ("pass2", _opts(rng, X0)),
        ("mid w=3 mean", _opts(rng, X0, "mid", window=3)),
        ("mid w=101 median exp2", _opts(rng, X0, "mid", window=101, center=1, apply_exp2=True)),
        ("log thr=0 w=1 none", dict(apply_log=True, window=1, center=0)),
        ("log bounds w=0 median", _opts(rng, X0, window=0, center=1)),
        ("no log bounds thr=2 mean exp2", _opts(rng, X0, apply_log=False, threshold=2.0, center=2)),
        ("window longer than every chromosome", _opts(rng, X0, window=2 * longest + 3)),
        ("smoothing only", dict(window=101)),
        ("centring only", dict(center=1)),
        ("stage D only", _opts(rng, X0, "stage_d")),
        ("stage D only, mid", _opts(rng, X0, "stage_d_mid")),
    ]
    cases = [Case(n, cs, cl, _no_minus_one_under_log(X0, o), o) for n, o in variants]
    sweep(api, monkeypatch, cases)
    DONE.add("options")


def test_column_placement(api, monkeypatch):
    """odd G (no column can take the bulk copy), an even G with column stride G + 1 (aligned and unaligned columns
    alternate inside a CTA's persistent loop and its prefetch of the next cell), an output stride ldy != G, and a column
    list in reverse order with repeats (pass 1's form)."""
    rng = np.random.default_rng(13)
    cases = []
    for lens in ([700, 1, 3, 501, 202, 1500, 97], [700, 1, 3, 501, 202, 1500, 98]):
        cs, cl = _layout(lens)
        G = int(cl.sum())
        X = _data(rng, G, 2 * _sm_count() + 3)
        cases.append(Case(f"G={G} ldx=G", cs, cl, X, _opts(rng, X)))
        cases.append(Case(f"G={G} ldx=G+1 ldy=G+3", cs, cl, X, _opts(rng, X), ldx=G + 1, ldy=G + 3))
        cols = np.concatenate([np.arange(X.shape[0])[::-1], [0, 0, 5, 2, 5]])
        cases.append(Case(f"G={G} reversed repeated cols", cs, cl, X, _opts(rng, X, "pass1"), cols=cols, ldx=G + 1))
    sweep(api, monkeypatch, cases)
    DONE.add("placement")


def test_cell_counts_around_the_grid(api, monkeypatch):
    """1, SMs - 1, SMs + 1, 2 SMs + 1 (two single-buffer CTAs per SM) and 3 SMs + 5 cells: the persistent loop's tails."""
    S = _sm_count()
    rng = np.random.default_rng(14)
    cs, cl = _layout([1000, 1, 333, 600, 2, 64] if EMULATED else [1000, 1, 333, 600, 2, 64, 1100, 99])
    G = int(cl.sum())
    cases = []
    for n in (1, S - 1, S + 1, 2 * S + 1, 3 * S + 5):
        X = _data(rng, G, n, special=n >= 4)
        cases.append(Case(f"{n} cells", cs, cl, X, _opts(rng, X)))
    sweep(api, monkeypatch, cases)
    DONE.add("cells")


def test_one_nan_sets_the_flag_on_every_variant(api, monkeypatch):
    rng = np.random.default_rng(15)
    cases = []
    for lens in ([900, 1, 3, 601, 202], [900, 1, 3, 601, 203]):       # bulk copies / element-wise loads
        cs, cl = _layout(lens)
        G = int(cl.sum())
        X = _data(rng, G, 3, special=False)
        X[1, G // 3] = np.nan
        cases.append(Case(f"NaN G={G}", cs, cl, X, _opts(rng, X)))
    try:
        for env in CONFIGS:
            _configure(api, monkeypatch, env)
            for c in cases:
                rc, _, flag, sel = c.run()
                assert rc == 0 and flag == 1 and sel[0] in (3, 4), (c.name, env, rc, flag, sel)
    finally:
        _configure(api, monkeypatch, {})
    DONE.add("nan")


@pytest.mark.skipif(EMULATED, reason="10 000 / 20 000 genes: too slow under the host emulation")
def test_alternating_layouts_in_one_process(api, monkeypatch):
    """10 000 genes (two-buffer kernel), 20 000 (single-buffer), 10 000 again, a different 10 000-gene layout: both families
    share the SLOT_SEGS scratch and the upload cache of the segment table; each result equals the first run of its layout."""
    _configure(api, monkeypatch, {})
    rng = np.random.default_rng(16)
    runs = []
    for G, lay in ((10000, "bench"), (20000, "bench"), (10000, "bench"), (10000, "other"), (20000, "bench"), (10000, "bench")):
        cs, cl = _bench_layout(G) if lay == "bench" else _layout([2500, 1, 1499, 3000, 2, 2998])
        X = _data(np.random.default_rng(G), G, 6)
        runs.append(((G, lay), Case(f"{G} {lay}", cs, cl, X, _opts(np.random.default_rng(G + 1), X))))
    first = {}
    for key, c in runs:
        rc, Y, flag, sel = c.run()
        assert rc == 0 and flag == 0
        if key in first:
            assert np.array_equal(Y.view(np.uint64), first[key].view(np.uint64)), key
        else:
            first[key] = Y
            want, bound = c.reference(sel[5], sel[1] // 32)
            r = cref.error_ratio(Y, want, bound)
            assert r <= 1.0, (key, r)
            _note(sel, r)
    DONE.add("alternating")


@pytest.mark.skipif(EMULATED, reason="Engine needs torch device tensors (tests/host/engine_emulated.py has these cases)")
def test_strided_torch_view_through_the_engine(api, monkeypatch):
    """Engine.cell_pipeline on X[:, :G] of a (C, G + 1) tensor: column stride G + 1, so aligned (bulk copy) and unaligned
    (element-wise) columns alternate; bit-identical to the same call on a contiguous copy, under every configuration."""
    torch = _torch()
    from infercnv_b200.device import Engine
    rng = np.random.default_rng(17)
    cs, cl = _layout([700, 1, 3, 501, 202, 1500, 98, 3000, 1994])
    G = int(cl.sum())
    C = 2 * _sm_count() + 5
    Xh = _data(rng, G, C)
    o = _opts(rng, Xh)
    want, _ = cref.cell_pipeline(Xh, cs, cl, L=1, NW=32, **o)
    wide = torch.zeros((C, G + 1), dtype=torch.float64, device="cuda")
    wide[:, :G] = torch.from_numpy(Xh).cuda()
    Xv = wide[:, :G]
    assert Xv.stride(0) == G + 1
    Xc = Xv.contiguous()
    b1 = tuple(torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (o["lo1"], o["hi1"], 0.5 * (o["lo1"] + o["hi1"])))
    b2 = tuple(torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (o["lo2"], o["hi2"], 0.5 * (o["lo2"] + o["hi2"])))
    try:
        for env in CONFIGS:
            _configure(api, monkeypatch, env)
            eng = Engine(0)
            out = []
            for X in (Xv, Xc):
                Y = torch.empty((C, G), dtype=torch.float64, device="cuda")
                flag = torch.zeros(1, dtype=torch.int32, device="cuda")
                eng.cell_pipeline(X, None, Y, cs, cl, True, b1, 3.0, 101, 1, b2, True, True, flag)
                assert int(flag.item()) == 0
                out.append(Y.cpu().numpy())
            sel = api.last_cell_kernel()
            assert np.array_equal(out[0].view(np.uint64), out[1].view(np.uint64)), (env, sel)
            _, bound = cref.cell_pipeline(Xh, cs, cl, L=sel[5], NW=sel[1] // 32, **o)
            r = cref.error_ratio(out[0], want, bound)
            assert r <= 1.0, (env, sel, r)
            _note(sel, r)
            k = f"element-wise load, cell_pipeline{sel[0]}_kernel"
            SPECIAL[k] = SPECIAL.get(k, 0) + 1
    finally:
        _configure(api, monkeypatch, {})
    DONE.add("engine")


def test_coverage_table():
    """One line per instantiation: cases run and the worst error as a fraction of the bound.  When the whole module ran on
    the H100, all 14 instantiations, both element-wise load paths and the refusal must be in it."""
    lines = [f"{_name(k + (0,)):42s} {v[0]:4d} cases   worst error / bound {v[1]:.2e}" for k, v in sorted(COVER.items())]
    lines += [f"{k:42s} {v:4d} cases" for k, v in sorted(SPECIAL.items())]
    print("\n[cell pipeline coverage]\n" + "\n".join(lines))
    everything = {"boundaries", "options", "placement", "cells", "nan", "alternating", "engine"} | {"layout_" + k for k in LAYOUTS}
    if not EMULATED and everything <= DONE:
        missing = ALL_INSTANTIATIONS - set(COVER)
        assert not missing, sorted(missing)
        assert {"refused with -4", "element-wise load, cell_pipeline3_kernel", "element-wise load, cell_pipeline4_kernel"} <= set(SPECIAL)
    if EMULATED and {"boundaries", "options", "placement", "cells"} <= DONE:
        reachable = {(3, nt, 1, pq, 0) for nt in (256, 512, 1024) for pq in (0, 1)} | {(4, 256, 4, 0, 0), (4, 512, 2, 0, 0), (4, 1024, 1, 0, 0)}
        assert reachable <= set(COVER), sorted(reachable - set(COVER))
