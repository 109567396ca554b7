"""`agglomerate` with waterz's histogram-quantile scoring functions, OneMinus<HistogramQuantileAffinity<...>>.

The rules are restated in oracle/agglomeration_quantile_oracle.py ("parity unpinned": waterz is not available).  On the CPU:
the scoring-function parser, known answers of the oracle decided by one rule each, the histogram region graph of
csrc/segmentation.cu compiled for the host behind the one-lane CUDA shim, and the native merge loop, all against the oracle.
On the GPU: the device histograms, DeviceChunk.agglomerate, the plugin and the CLI against the oracle, and a larger run."""
import ctypes as C

import numpy as np
import pytest

import host_emulation
from oracle import agglomeration_oracle as A
from oracle import agglomeration_quantile_oracle as H

LOW, HIGH = 0.001, 0.9999
HQ50 = 'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 256, false>>'
HQ50_INITMAX = 'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 256, true>>'
HQ_ODD = 'OneMinus<HistogramQuantileAffinity<RegionGraphType, 37, ScoreValue, 13>>'   # I omitted: true


def _affinities(seed, shape, kind):
    """kind: 0 random float32, 1 quantised to quarters (ties), 2 smooth (like a network output), 3 NaNs and values outside
    [0, 1] sprinkled into a smooth map."""
    rng = np.random.default_rng(seed)
    a = rng.random((3,) + tuple(shape)).astype(np.float32)
    if kind == 1:
        a = (np.round(a * 4) / 4 * 0.9).astype(np.float32)
    elif kind >= 2:
        from scipy import ndimage
        a = ndimage.gaussian_filter(rng.standard_normal(a.shape), sigma=(0, 1.0, 2.0, 2.0))
        a = (1.0 / (1.0 + np.exp(-4.0 * a / a.std()))).astype(np.float32)
        if kind == 3:
            r = rng.random(a.shape)
            a[r < 0.03] = np.nan
            a[(r >= 0.03) & (r < 0.06)] = 1.5
            a[(r >= 0.06) & (r < 0.09)] = -0.25
    return a


# ------------------------------------------------------------------------------------------------------------
# the scoring-function string
# ------------------------------------------------------------------------------------------------------------
def test_parser_accepts_the_family_and_refuses_everything_else():
    from chunkflow_b200.chunk.device import HistogramQuantile, parse_scoring_function as parse
    assert parse('OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>') is None
    assert parse(' OneMinus< MeanAffinity<RegionGraphType,ScoreValue> > ') is None
    assert parse(HQ50) == HistogramQuantile(50, 256, False)
    assert parse(HQ50_INITMAX) == HistogramQuantile(50, 256, True)
    assert parse('OneMinus<HistogramQuantileAffinity<RegionGraphType,75,ScoreValue,100>>') == HistogramQuantile(75, 100, True)
    assert parse('OneMinus < HistogramQuantileAffinity <\tRegionGraphType , 0 ,\nScoreValue , 2 , true > >') == \
        HistogramQuantile(0, 2, True)
    assert parse('OneMinus<HistogramQuantileAffinity<RegionGraphType, 100, ScoreValue, 256, false>>') == \
        HistogramQuantile(100, 256, False)
    for other in ('OneMinus<MaxAffinity<RegionGraphType, ScoreValue>>',
                  'OneMinus<QuantileAffinity<RegionGraphType, 50, ScoreValue>>',
                  'OneMinus<MeanMaxKAffinity<RegionGraphType, 10, ScoreValue>>',
                  'Multiply<OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>, MinSize<SizeType, ScoreValue>>',
                  'HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 256, false>',
                  'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue>>',
                  'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 256, false, 1>>',
                  'OneMinus<HistogramQuantileAffinity<RegionGraphType, 5.0, ScoreValue, 256>>', '', None):
        with pytest.raises(NotImplementedError):
            parse(other)
    for bad in ('OneMinus<HistogramQuantileAffinity<RegionGraphType, 101, ScoreValue, 256>>',
                'OneMinus<HistogramQuantileAffinity<RegionGraphType, -1, ScoreValue, 256>>',
                'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 1>>',
                'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 257>>',
                'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 256, True>>',
                'OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 256, 1>>'):
        with pytest.raises(ValueError):
            parse(bad)


def test_plugin_and_cli_refuse_before_touching_the_gpu():
    from click.testing import CliRunner
    from chunkflow_b200 import Chunk
    from chunkflow_b200.flow import cli
    from chunkflow_b200.plugins import agglomerate
    affs = Chunk(np.zeros((3, 2, 4, 4), np.float32))
    with pytest.raises(NotImplementedError):
        agglomerate.execute(affs, scoring_function='OneMinus<MaxAffinity<RegionGraphType, ScoreValue>>')
    with pytest.raises(ValueError):
        agglomerate.execute(affs, scoring_function='OneMinus<HistogramQuantileAffinity<RegionGraphType, 50, ScoreValue, 300>>')
    opts = {o for p in cli.agglomerate.params for o in p.opts}
    assert "--scoring-function" in opts
    assert {p.name: p.default for p in cli.agglomerate.params}["scoring_function"] == agglomerate.SCORING_FUNCTION
    res = CliRunner().invoke(cli.main, ["create-chunk", "agglomerate", "--scoring-function",
                                        'OneMinus<MaxAffinity<RegionGraphType, ScoreValue>>'], standalone_mode=False)
    assert isinstance(res.exception, NotImplementedError)


# ------------------------------------------------------------------------------------------------------------
# the oracle: known answers, one rule each
# ------------------------------------------------------------------------------------------------------------
def _graph(edges, B):
    """edges: [(u, v, {bin: count}, max)] -> the arrays of a histogram region graph."""
    u = np.array([e[0] for e in edges], np.uint32)
    v = np.array([e[1] for e in edges], np.uint32)
    runs = [sorted(e[2].items()) for e in edges]
    off = np.cumsum([0] + [len(r) for r in runs]).astype(np.uint64)
    bins = np.array([b for r in runs for b, _ in r], np.uint8)
    cnt = np.array([c for r in runs for _, c in r], np.uint32)
    mx = np.array([e[3] for e in edges], np.float32)
    return u, v, off, bins, cnt, mx


def _both(num_nodes, edges, thr, Q, B, I):
    """oracle result, checked against the native loop (same arrays)."""
    from chunkflow_b200 import _native
    g = _graph(edges, B)
    ref = H.agglomerate_edges_quantile(num_nodes, *g, thr, Q, B, I)
    got = _native.agglomerate_quantile_host(num_nodes, *g, thr, Q, B, I)
    assert np.array_equal(got, ref), (got, ref)
    return ref.tolist()


def test_oracle_bins_clamp_nan_and_range():
    b, c = H.affinity_bins(np.array([1.0, 0.99999994, 0.5, 0.2499, 0.0, -0.3, 2.0, np.nan, -0.0], np.float32), 4)
    assert b.tolist() == [3, 3, 2, 0, 0, 0, 3, 0, 0]                     # a * B = B lands in the last bin
    assert c.tolist() == [1.0, np.float32(0.99999994), 0.5, np.float32(0.2499), 0.0, 0.0, 1.0, 0.0, 0.0]
    assert H.affinity_bins(np.array([0.5, 0.999], np.float32), 256)[0].tolist() == [128, 255]
    # a row 1 2 1 2: three x faces between fragments 1 and 2 with NaN, 1.5 and -0.2; the y/z channels have no faces
    a = np.zeros((3, 1, 1, 4), np.float32)
    a[2, 0, 0, 1:] = (np.nan, 1.5, -0.2)
    u, v, off, bins, cnt, mx = H.region_graph_histograms(a, np.array([[[1, 2, 1, 2]]]), 4, True)
    assert (u.tolist(), v.tolist(), off.tolist(), bins.tolist(), cnt.tolist(), mx.tolist()) == ([1], [2], [0, 2], [0, 3], [2, 1], [1.0])
    assert H.region_graph_histograms(a, np.array([[[1, 2, 1, 2]]]), 4, False)[5] is None


def test_oracle_pivot_at_small_n_and_the_extreme_quantiles():
    # two faces, bins 0 and 3 of 4: Q = 50 -> pivot min(1 + 1, 2) = 2 -> bin 3 (score 0.125); Q = 49 -> pivot 1 -> bin 0 (0.875)
    e = [(1, 2, {0: 1, 3: 1}, 0.9)]
    assert H.quantile_score(np.array([1, 0, 0, 1]), 50, 4) == 0.125
    assert H.quantile_score(np.array([1, 0, 0, 1]), 49, 4) == 0.875
    assert _both(3, e, 0.5, 50, 4, False) == [0, 1, 1]
    assert _both(3, e, 0.5, 49, 4, False) == [0, 1, 2]
    # one face: every quantile is its bin
    assert _both(3, [(1, 2, {2: 1}, 0.6)], 0.4, 0, 4, False) == [0, 1, 1]
    assert _both(3, [(1, 2, {2: 1}, 0.6)], 0.375, 100, 4, False) == [0, 1, 2]   # 0.375 is not below 0.375
    # Q = 0 takes the lowest non-empty bin, Q = 100 the highest (pivot = n, not n + 1)
    e = [(1, 2, {1: 3, 3: 1}, 0.9)]
    assert H.quantile_score(np.array([0, 3, 0, 1]), 0, 4) == 0.625 and H.quantile_score(np.array([0, 3, 0, 1]), 100, 4) == 0.125
    assert _both(3, e, 0.5, 0, 4, False) == [0, 1, 2]
    assert _both(3, e, 0.5, 100, 4, False) == [0, 1, 1]


def test_oracle_init_with_max_before_and_after_pooling():
    # (1,2) merges on its maximum; then (1,3) and (2,3) pool and score from the pooled histogram {0: 1, 1: 1}: bin 1, 0.625
    e = [(1, 2, {0: 5}, 0.9), (1, 3, {0: 1}, 0.8), (2, 3, {1: 1}, 0.7)]
    assert _both(4, e, 0.5, 50, 4, True) == [0, 1, 1, 3]        # 0.625 >= 0.5 although both maxima scored below it
    assert _both(4, e, 0.7, 50, 4, True) == [0, 1, 1, 1]
    assert _both(4, e, 0.5, 50, 4, False) == [0, 1, 2, 3]       # without I every score comes from the histogram
    # a MOVED edge keeps its max score: (2,3) alone moves to cluster 1 and still scores 1 - 0.7
    e = [(1, 2, {0: 5}, 0.9), (2, 3, {0: 1}, 0.7)]
    assert _both(4, e, 0.35, 50, 4, True) == [0, 1, 1, 1]


def test_pooled_edge_below_the_edge_being_merged():
    """I = true: (1,2) scores 1 - 0.5 and merges; (1,3) and (2,3), whose faces all lie in bin 128 of 256 (value 0.50195),
    pool to 1 - 0.50195 < 0.5 -- below the edge just merged, so a queue that only ever moves forward would lose it."""
    e = [(1, 2, {128: 1}, 0.5), (1, 3, {128: 1}, 0.5), (2, 3, {128: 1}, 0.5)]
    assert H.quantile_score(np.bincount([128, 128], minlength=256), 50, 256) < 0.5
    assert _both(4, e, 0.5001, 50, 256, True) == [0, 1, 1, 1]
    assert _both(4, e, 0.5, 50, 256, True) == [0, 1, 2, 3]        # 0.5 itself does not merge
    # with more of the graph around it: (3,4) at 1 - 0.501 merges first, then the same cascade
    e.append((3, 4, {128: 4}, 0.501))
    assert _both(5, e, 0.5001, 50, 256, True) == [0, 1, 1, 1, 1]


def test_rule_6_anchor_decides_the_order():
    """After (1,2) merges, (1,5) [1 face, bin 1] and (2,5) [3 faces, bin 2] pool to the median bin 2 -- 0.375, the score of
    (2,5) -- and keep (2,5)'s anchor.  (1,6), also at 0.375, has the anchor between (1,5) and (2,5), so it merges first; then
    cluster 1's edge to 5 pools with (5,6) and rises to 0.875.  The smaller-anchor rule of the mean would merge 5 instead."""
    e = [(1, 2, {3: 1}, 0.0), (1, 5, {1: 1}, 0.0), (2, 5, {2: 3}, 0.0), (1, 6, {2: 1}, 0.0), (5, 6, {0: 10}, 0.0)]
    assert _both(7, e, 0.5, 50, 4, False) == [0, 1, 1, 3, 4, 5, 1]


# ------------------------------------------------------------------------------------------------------------
# the histogram region graph of segmentation.cu on the host (one-lane CUDA shim)
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("rg_hist", tmp_path_factory)
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    lib.cfb_region_graph_hist_workspace.argtypes = [i64]
    lib.cfb_region_graph_hist_workspace.restype = i64
    lib.cfb_region_graph_hist_device.argtypes = [vp, i32, vp, i64, i64, i64, i32, vp, i64, C.POINTER(i64), C.POINTER(i64), vp]
    lib.cfb_region_graph_hist_read.argtypes = [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, vp]
    return lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _emu_hist(lib, affs, flip, frag, B, slots):
    """(rc, u, v, offsets, bins, counts, maxima) of the emulated passes and read; rc = -6 when a table is too small."""
    affs, frag = np.ascontiguousarray(affs, np.float32), np.ascontiguousarray(frag, np.uint32)
    z, y, x = frag.shape
    work = np.zeros(lib.cfb_region_graph_hist_workspace(slots) // 8 + 1, np.uint64)
    n, nh = C.c_int64(), C.c_int64()
    rc = lib.cfb_region_graph_hist_device(_p(affs), flip, _p(frag), z, y, x, B, _p(work), slots, C.byref(n), C.byref(nh), None)
    if rc != 0:
        return (rc,)
    n, nh = n.value, nh.value
    u, v, mx = np.empty(n, np.uint32), np.empty(n, np.uint32), np.empty(n, np.float32)
    off, b, c = np.empty(n + 1, np.uint64), np.empty(nh, np.uint8), np.empty(nh, np.uint32)
    assert lib.cfb_region_graph_hist_read(_p(work), slots, n, nh, _p(u), _p(v), _p(off), _p(b), _p(c), _p(mx), None) == 0, \
        lib.cfb_last_error()
    return 0, u, v, off, b, c, mx


def _same_graph(got, ref):
    for g, r, name in zip(got, ref, ("u", "v", "offsets", "bins", "counts", "maxima")):
        assert g.dtype == r.dtype and np.array_equal(g, r), name


def test_emulated_histogram_passes_against_the_oracle(emu):
    from chunkflow_b200._native import ERR_CAPACITY
    rng = np.random.default_rng(3)
    for trial in range(16):
        shape = tuple(int(s) for s in rng.integers(2, 12, 3))
        kind = trial % 4
        a = _affinities(200 + trial, shape, kind)                  # waterz's order z, y, x
        if trial % 3 == 2:                                        # fragments handed in: blocks, some background
            frag = (np.arange(a[0].size).reshape(shape) // 3 % 7).astype(np.uint32)
        else:
            frag = A.watershed(np.nan_to_num(a, nan=0.5), LOW, HIGH)
        B = (2, 100, 256, 13)[trial % 4]
        ref = H.region_graph_histograms(a, frag, B, True)
        slots = 1 << max(4, int(np.ceil(np.log2(2 * len(ref[0]) + 1))))
        got = _emu_hist(emu, a, 0, frag, B, 4 * slots)
        assert got[0] == 0
        _same_graph(got[1:], ref)
        flipped = _emu_hist(emu, np.ascontiguousarray(a[::-1]), 1, frag, B, 4 * slots)   # chunkflow's order, read in reverse
        _same_graph(flipped[1:], ref)
        # a pair table that cannot hold the pairs, and one that holds them while the bin table does not
        if len(ref[0]) > 2:
            assert _emu_hist(emu, a, 0, frag, B, 2) == (ERR_CAPACITY,)
    a = _affinities(7, (6, 20, 20), 0)
    frag = np.zeros((6, 20, 20), np.uint32)
    frag[:, :, :10], frag[:, :, 10:] = 1, 2                       # one pair, 120 faces over up to 256 bins
    assert _emu_hist(emu, a, 0, frag, 256, 2) == (ERR_CAPACITY,)   # pair table of 2 slots, bin table of 4
    got = _emu_hist(emu, a, 0, frag, 256, 256)
    assert got[0] == 0 and len(got[4]) > 8
    _same_graph(got[1:], H.region_graph_histograms(a, frag, 256, True))


def test_whole_operator_with_emulated_passes_and_the_native_loop(emu):
    """watershed (oracle) -> histogram region graph (emulated kernels) -> cfb_agglomerate_quantile_host == the oracle's plugin."""
    from chunkflow_b200 import _native
    for seed, shape, kind, thr, (Q, B, I) in ((0, (6, 10, 12), 2, 0.5, (50, 256, False)), (1, (8, 12, 12), 2, 0.4, (50, 256, True)),
                                              (2, (5, 9, 9), 1, 0.8, (37, 13, True)), (3, (6, 10, 10), 3, 0.6, (75, 100, False))):
        a = _affinities(seed, shape, kind)                        # chunkflow's order x, y, z
        frag = A.watershed(np.ascontiguousarray(a[::-1]), LOW, HIGH)
        _, u, v, off, b, c, mx = _emu_hist(emu, a, 1, frag, B, 1 << 14)
        root = _native.agglomerate_quantile_host(int(frag.max()) + 1, u, v, off, b, c, mx, thr, Q, B, I)
        assert np.array_equal(root[frag].astype(np.uint64), H.agglomerate(a, thr, Q, B, I)), (seed, kind)


# ------------------------------------------------------------------------------------------------------------
# the native merge loop (no GPU involved)
# ------------------------------------------------------------------------------------------------------------
def _tied_graph(rng, B):
    """A random sparse graph whose faces sit on a few bin centres (ties everywhere); the maxima are those centres."""
    n = int(rng.integers(2, 60))
    pairs = set()
    for _ in range(int(rng.integers(0, n * 3))):
        p, q = (int(t) for t in rng.integers(1, n, 2))
        if p != q:
            pairs.add((min(p, q), max(p, q)))
    levels = rng.choice(B, size=min(B, int(rng.choice([2, 3, 5]))), replace=False)
    edges = []
    for p, q in sorted(pairs):
        faces = rng.choice(levels, size=int(rng.integers(1, 7)))
        hist = {int(b): int(k) for b, k in zip(*np.unique(faces, return_counts=True))}
        edges.append((p, q, hist, float(np.float32((faces.max() + 0.5) / B))))
    return n, edges


@pytest.mark.parametrize("mode,threads,grain", [("0", "1", "2048"), ("1", "4", "2048"), ("2", "5", "3"), ("2", "8", "1")])
def test_native_quantile_loop_fuzz_against_the_oracle(monkeypatch, mode, threads, grain):
    """Heavy ties; Q in {0, 10, 50, 75, 100}, B in {2, 100, 256}, both I, thresholds inside and at the ends of the range.
    The rounds do not run for this family, so every knob must leave the result as it is."""
    from chunkflow_b200 import _native
    monkeypatch.setenv("CFB_AGGLOMERATE_MODE", mode)
    monkeypatch.setenv("CFB_AGGLOMERATE_THREADS", threads)
    monkeypatch.setenv("CFB_AGGLOMERATE_GRAIN", grain)
    rng = np.random.default_rng(11)
    for t in range(60):
        Q, B, I = (0, 10, 50, 75, 100)[t % 5], (2, 100, 256)[t % 3], bool(t % 2)
        n, edges = _tied_graph(rng, B)
        g = _graph(edges, B)
        for thr in (float(rng.random()), 0.0, 0.5, 1.0, float("inf")):
            ref = H.agglomerate_edges_quantile(n, *g, thr, Q, B, I)
            assert np.array_equal(_native.agglomerate_quantile_host(n, *g, thr, Q, B, I), ref), (t, thr, Q, B, I)
            assert np.array_equal(ref[ref], ref) and (ref <= np.arange(n)).all()


@pytest.mark.parametrize("mode", ["0", "1", "2"])
def test_native_quantile_loop_on_region_graphs(monkeypatch, mode):
    """Region graphs of watershed fragments (more than 4096 edges in the last one) with the oracle's histograms."""
    from chunkflow_b200 import _native
    monkeypatch.setenv("CFB_AGGLOMERATE_MODE", mode)
    for trial, (shape, kind, thr, (Q, B, I)) in enumerate((((6, 10, 12), 0, 0.5, (50, 256, False)), ((8, 12, 12), 2, 0.3, (50, 256, True)),
                                                           ((5, 9, 9), 1, 0.8, (10, 2, True)), ((10, 30, 30), 0, 0.45, (75, 100, True)))):
        a = _affinities(trial, shape, kind)
        frag = A.watershed(a, LOW, HIGH)
        g = H.region_graph_histograms(a, frag, B, I)
        n = int(frag.max()) + 1
        assert np.array_equal(_native.agglomerate_quantile_host(n, *g, thr, Q, B, I), H.agglomerate_edges_quantile(n, *g, thr, Q, B, I))


def test_native_quantile_loop_refuses_malformed_input():
    from chunkflow_b200 import _native
    g = _graph([(1, 2, {0: 1, 3: 2}, 0.5)], 4)
    assert _native.agglomerate_quantile_host(3, [], [], [0], [], [], None, 0.5, 50, 4, False).tolist() == [0, 1, 2]
    for args in ((3, *g, 0.5, 101, 4, False), (3, *g, 0.5, 50, 1, False), (3, *g, 0.5, 50, 3, False),   # bin 3 >= B
                 (2, *g, 0.5, 50, 4, False),                                                            # id outside the nodes
                 (3, g[0], g[1], g[2], g[3][::-1].copy(), g[4], g[5], 0.5, 50, 4, False),               # bins out of order
                 (3, g[0], g[1], g[2], g[3], np.zeros(2, np.uint32), g[5], 0.5, 50, 4, False),           # zero counts
                 (3, g[0], g[1], g[2], g[3], g[4], np.array([np.nan], np.float32), 0.5, 50, 4, True),   # a NaN maximum
                 (3, *_graph([(1, 2, {0: 1}, 0.5), (2, 1, {1: 1}, 0.5)], 4), 0.5, 50, 4, False)):      # duplicate edge
        with pytest.raises(_native.NativeError):
            _native.agglomerate_quantile_host(*args)


# ------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_histogram_region_graph_against_the_oracle():
    import torch
    from chunkflow_b200.chunk.device import DeviceChunk
    for seed, shape, kind, B in ((0, (17, 40, 53), 0, 256), (1, (9, 33, 64), 1, 2), (2, (24, 48, 48), 2, 100), (3, (12, 30, 31), 3, 13),
                                 (4, (1, 1, 7), 0, 256), (5, (16, 64, 64), 2, 256)):
        a = _affinities(seed, shape, kind)                         # waterz order z, y, x
        ref_frag = A.watershed(np.nan_to_num(a, nan=0.5), LOW, HIGH)
        ref = H.region_graph_histograms(a, ref_frag, B, True)
        for flip in (False, True):
            stored = np.ascontiguousarray(a[::-1]) if flip else a
            dev = DeviceChunk(torch.from_numpy(stored).cuda(), layer_type="affinity_map")
            frag = DeviceChunk(torch.from_numpy(ref_frag.astype(np.int32)).cuda(), layer_type="segmentation")
            got = dev.region_graph(frag, flip_channel=flip, histogram_bins=B)
            _same_graph(got, ref)
    # many bins per pair: the bin table outgrows its first size and is rebuilt larger
    a = _affinities(8, (32, 64, 64), 0)
    f = np.zeros((32, 64, 64), np.int32)
    f[:, :, 32:] = 1
    f[:, 32:, :] += 2
    f += 1
    dev = DeviceChunk(torch.from_numpy(a).cuda(), layer_type="affinity_map")
    got = dev.region_graph(DeviceChunk(torch.from_numpy(f).cuda(), layer_type="segmentation"), flip_channel=False, num_fragments=4,
                           histogram_bins=256)
    _same_graph(got, H.region_graph_histograms(a, f, 256, True))


def _maps():
    return [(0, (16, 64, 64), 2, 0.5), (1, (24, 64, 64), 2, 0.35), (2, (32, 64, 64), 3, 0.6)]


@pytest.mark.gpu
def test_device_plugin_and_deviceChunk_against_the_oracle():
    import torch
    from chunkflow_b200 import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk, parse_scoring_function
    from chunkflow_b200.plugins import agglomerate
    for (seed, shape, kind, thr), sf in zip(_maps(), (HQ50, HQ50_INITMAX, HQ_ODD)):
        Q, B, I = parse_scoring_function(sf)
        a = _affinities(seed, shape, kind)                         # chunkflow's order x, y, z: the plugin flips
        ref = H.agglomerate(a, thr, Q, B, I)
        out = agglomerate.execute(Chunk(a, voxel_offset=(5, 6, 7), voxel_size=(40, 4, 4)), threshold=thr, scoring_function=sf)[0]
        assert out.array.dtype == np.uint64 and tuple(out.voxel_offset) == (5, 6, 7)
        assert np.array_equal(out.array, ref), (seed, sf)
        frag = A.watershed(np.flip(a, 0), 0.3, 0.8)                # fragments handed in
        ref2 = H.agglomerate(a, thr, Q, B, I, fragments=frag)
        assert np.array_equal(agglomerate.execute(Chunk(a), fragments=frag.astype(np.uint64), threshold=thr, scoring_function=sf)[0].array, ref2)
        dev = DeviceChunk(torch.from_numpy(a).cuda(), layer_type="affinity_map")
        seg = dev.agglomerate(threshold=thr, scoring_function=sf)
        assert np.array_equal(seg.tensor.cpu().numpy().view(np.uint32).astype(np.uint64), ref)
        f = DeviceChunk(torch.from_numpy(frag.astype(np.int32)).cuda(), layer_type="segmentation")
        seg2 = dev.agglomerate(threshold=thr, fragments=f, scoring_function=sf)
        assert np.array_equal(seg2.tensor.cpu().numpy().view(np.uint32).astype(np.uint64), ref2)


@pytest.mark.gpu
def test_device_cli_on_host_and_device_chunks_against_the_oracle():
    from click.testing import CliRunner
    from chunkflow_b200 import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk, parse_scoring_function
    from chunkflow_b200.flow.cli import main, operator
    seed, shape, kind, thr = _maps()[0]
    a = _affinities(seed, shape, kind)
    seen = {}

    @main.command("capture-quantile-test")
    @operator
    def capture(tasks):
        for task in tasks:
            seen.update(task)
            yield task
    try:
        @main.command("load-quantile-test")
        @operator
        def load(tasks):
            for task in tasks:
                task["affs"] = Chunk(a.copy(), voxel_offset=(2, 4, 6))
                yield task
        args = ["load-quantile-test"]
        for i, sf in enumerate((HQ50, HQ50_INITMAX, HQ_ODD)):
            args += ["agglomerate", "-i", "affs", "-o", f"seg{i}", "-t", str(thr), "--scoring-function", sf]
        args += ["to-device", "-i", "affs", "-o", "daffs", "agglomerate", "-i", "daffs", "-o", "dseg", "-t", str(thr),
                 "--scoring-function", HQ50_INITMAX, "to-host", "-i", "dseg", "-o", "hseg", "capture-quantile-test"]
        r = CliRunner().invoke(main, args, catch_exceptions=False)
        assert r.exit_code == 0, r.output
    finally:
        main.commands.pop("capture-quantile-test", None)
        main.commands.pop("load-quantile-test", None)
    for i, sf in enumerate((HQ50, HQ50_INITMAX, HQ_ODD)):
        assert isinstance(seen[f"seg{i}"], Chunk)
        assert np.array_equal(np.asarray(seen[f"seg{i}"].array).astype(np.uint64), H.agglomerate(a, thr, *parse_scoring_function(sf))), sf
    assert isinstance(seen["dseg"], DeviceChunk)
    assert np.array_equal(np.asarray(seen["hseg"].array).astype(np.uint64), H.agglomerate(a, thr, 50, 256, True))


@pytest.mark.gpu
def test_quantile_agglomerate_on_a_larger_volume():
    """3 x 64 x 256 x 256: the surviving ids are fragment ids (the smallest of each cluster), and a higher threshold merges no
    fewer regions."""
    import torch
    from chunkflow_b200.chunk.device import DeviceChunk
    a = _affinities(21, (64, 256, 256), 2)
    dev = DeviceChunk(torch.from_numpy(a).cuda(), layer_type="affinity_map")
    frag = dev.watershed(LOW, HIGH)
    f = frag.tensor.cpu().numpy().view(np.uint32)
    for sf in (HQ50, HQ50_INITMAX):
        segs = []
        for thr in (0.3, 0.6):
            seg = dev.agglomerate(threshold=thr, fragments=frag, scoring_function=sf).tensor.cpu().numpy().view(np.uint32)
            assert np.array_equal(seg == 0, f == 0) and (seg <= f).all()
            assert set(np.unique(seg).tolist()) <= set(np.unique(f).tolist())
            pairs = np.unique(np.stack([f.ravel(), seg.ravel()]), axis=1)
            assert len(pairs[0]) == frag.num_components + 1      # every fragment goes to exactly one segment
            segs.append(len(np.unique(seg)))
        assert segs[1] <= segs[0] < frag.num_components + 1
