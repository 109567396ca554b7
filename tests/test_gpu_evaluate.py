"""`evaluate-segmentation` on the H100 (csrc/evaluate.cu through the C ABI, DeviceChunk.evaluate, Segmentation.evaluate and
the CLI) against the golden vectors of the real reference and the numpy oracle (oracle/evaluation_oracle.py)."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

from oracle import evaluation_oracle as EV

pytestmark = pytest.mark.gpu

SCORES = ("rand_index", "adjusted_rand_index", "variation_of_information", "fowlkes_mallows_index")


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


def dev(torch, arr):
    from chunkflow_b200.chunk.segmentation import _device_labels
    return _device_labels(np.asarray(arr), "cuda:0")


@pytest.fixture(scope="module")
def gold():
    from test_evaluate_oracle import GOLDEN
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def same_bits(a, b):
    return np.float64(a).tobytes() == np.float64(b).tobytes()


def test_device_against_golden(torch, gold):
    from test_evaluate_oracle import assert_scores_match, golden_cases
    for name in golden_cases(gold):
        s, g = dev(torch, gold[f"{name}/seg"]), dev(torch, gold[f"{name}/gt"])
        seg_ids, gt_ids, counts = s.contingency_table(g)
        np.testing.assert_array_equal(np.stack([seg_ids, gt_ids, counts.astype(np.uint64)], 1), gold[f"{name}/table"], err_msg=name)
        stats = s.evaluate_statistics(g, tuple(gold[f"{name}/scores"][:, 0]))
        for row, st in zip(gold[f"{name}/scores"], stats):
            assert_scores_match(dict(st, edit_distance=(st["false_merges"], st["false_splits"])), row)


def test_segmentation_evaluate_prints_and_returns_like_the_reference(torch, gold):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.segmentation import Segmentation
    from test_evaluate_oracle import assert_scores_match
    for name in ("random_u32", "blobs_int64", "one_label"):
        buf = io.StringIO()
        with redirect_stdout(buf):
            r = Segmentation(Chunk(gold[f"{name}/seg"])).evaluate(Chunk(gold[f"{name}/gt"]), size_threshold=1000)
        assert sorted(r) == sorted(SCORES + ("edit_distance",))
        assert_scores_match(r, gold[f"{name}/scores"][2])
        assert buf.getvalue() == str(gold[f"{name}/printed"][2])


def random_pair(rng, shape, pool_size=40):
    special = np.array([0, 2 ** 63 + 5, 2 ** 64 - 1, 1], np.uint64)
    pool = np.unique(np.concatenate([special, rng.integers(0, 2 ** 64, pool_size, dtype=np.uint64)]))
    assert pool.dtype == np.uint64 and np.isin(special, pool).all()
    seg = pool[rng.integers(0, pool.size, shape)]
    gt = pool[rng.integers(0, pool.size, shape)]
    seg[:, :, : shape[2] // 3] = seg[:, :, :1]   # runs of equal pairs along x
    gt[:, :, : shape[2] // 3] = gt[:, :, :1]
    return seg, gt


@pytest.mark.parametrize("seed", range(4))
def test_device_table_and_statistics_equal_the_oracle(torch, seed):
    rng = np.random.default_rng(seed)
    seg, gt = random_pair(rng, (7, 33, 65))
    s, g = dev(torch, seg), dev(torch, gt)
    ids_s, ids_g, c = s.contingency_table(g)
    os_, og, oc = EV.contingency_triples(seg, gt)
    np.testing.assert_array_equal(ids_s, os_); np.testing.assert_array_equal(ids_g, og); np.testing.assert_array_equal(c, oc)
    st = s.evaluate_statistics(g, (3,))[0]
    want = EV.statistics(os_, og, oc, 3)
    for k, v in want.items():
        assert st[k] == (pytest.approx(v, rel=1e-14) if k.startswith("xlog") else v), k
    # uint8 / uint32 inputs
    seg8 = (seg % np.uint64(7)).astype(np.uint8)
    gt32 = (gt >> np.uint64(40)).astype(np.uint32)
    ids_s, ids_g, c = dev(torch, seg8).contingency_table(dev(torch, gt32))
    os_, og, oc = EV.contingency_triples(seg8, gt32)
    np.testing.assert_array_equal(ids_s, os_); np.testing.assert_array_equal(ids_g, og); np.testing.assert_array_equal(c, oc)


def test_relabelling_gives_bitwise_identical_scores(torch):
    rng = np.random.default_rng(11)
    seg = rng.integers(0, 300, (16, 64, 64)); seg[:, :, 10:40] = seg[:, :, 10:11]
    gt = rng.integers(0, 200, (16, 64, 64)); gt[:, 5:30] = gt[:, 5:6]
    base = dev(torch, seg.astype(np.uint32)).evaluate_statistics(dev(torch, gt.astype(np.uint32)), (0, 10, 1000))
    for trial in range(2):
        # a random bijection onto wide ids (2^64 - 1 and ids >= 2^63 included) that keeps 0, the ignored label, at 0
        ids = rng.permutation(np.unique(rng.integers(1, 2 ** 64 - 1, 600, dtype=np.uint64)))[:299]
        ids = np.concatenate([np.array([0, 2 ** 64 - 1], np.uint64), ids])
        assert np.unique(ids).size == 301 and (ids >= 2 ** 63).sum() > 100
        other = dev(torch, ids[seg]).evaluate_statistics(dev(torch, ids[gt]), (0, 10, 1000))
        for a, b in zip(base, other):
            for k in SCORES + ("false_merges", "false_splits"):
                assert same_bits(a[k], b[k]), (trial, k, a[k], b[k])


def test_swap_symmetry(torch):
    rng = np.random.default_rng(3)
    seg, gt = random_pair(rng, (9, 40, 40))
    a = dev(torch, seg).evaluate(dev(torch, gt))
    b = dev(torch, gt).evaluate(dev(torch, seg))
    for k in SCORES:
        assert same_bits(a[k], b[k]), k


def test_two_runs_are_bitwise_equal(torch):
    rng = np.random.default_rng(4)
    seg, gt = random_pair(rng, (32, 128, 128), pool_size=3000)
    s, g = dev(torch, seg), dev(torch, gt)
    r1 = s.evaluate_statistics(g, (0, 10, 1000))
    r2 = s.evaluate_statistics(g, (0, 10, 1000))
    for a, b in zip(r1, r2):
        assert all(same_bits(a[k], b[k]) for k in a), (a, b)


def test_capacity_retry_from_a_tiny_table(torch):
    rng = np.random.default_rng(5)
    seg, gt = random_pair(rng, (8, 32, 32), pool_size=200)
    s, g = dev(torch, seg), dev(torch, gt)
    from chunkflow_b200 import _native
    work = torch.empty(_native.evaluate_workspace(32), dtype=torch.uint8, device="cuda:0")
    with pytest.raises(_native.NativeError) as err:
        _native.contingency_device(s.tensor.data_ptr(), _native.DTYPE_U64, g.tensor.data_ptr(), _native.DTYPE_U64, seg.shape,
                                   work.data_ptr(), 32)
    assert err.value.code == _native.ERR_CAPACITY
    ids_s, ids_g, c = s.contingency_table(g, table_slots=32)
    os_, og, oc = EV.contingency_triples(seg, gt)
    np.testing.assert_array_equal(ids_s, os_); np.testing.assert_array_equal(ids_g, og); np.testing.assert_array_equal(c, oc)
    r = s.evaluate(g, 10, table_slots=32)
    w = EV.evaluate(seg, gt, 10)
    for k in ("rand_index", "adjusted_rand_index", "fowlkes_mallows_index"):
        assert same_bits(r[k], w[k]), k
    assert r["edit_distance"] == w["edit_distance"]


def test_degenerate_cases_return_nan(torch):
    z = np.zeros((4, 5, 6), np.uint64)
    r = dev(torch, z).evaluate(dev(torch, z))
    np.testing.assert_equal([r[k] for k in SCORES], [1.0, np.nan, np.nan, 1.0]); assert r["edit_distance"] == (0.0, 0.0)
    one = np.full((4, 5, 6), 7, np.uint32)
    r = dev(torch, one).evaluate(dev(torch, one))
    np.testing.assert_equal([r[k] for k in SCORES], [1.0, np.nan, 0.0, 1.0]); assert r["edit_distance"] == (-1.0, 0.0)
    d = np.arange(1, 61, dtype=np.uint32).reshape(3, 4, 5)
    r = dev(torch, d).evaluate(dev(torch, d), size_threshold=0)
    np.testing.assert_equal([r[k] for k in SCORES], [1.0, np.nan, 0.0, np.nan]); assert r["edit_distance"] == (0.0, 0.0)


def test_large_volume_agrees_with_the_oracle(torch):
    """256 x 512 x 512 with about 10^5 distinct pairs: coherent blocks of one pair each, plus a salt of random pairs."""
    rng = np.random.default_rng(6)
    shape = (256, 512, 512)
    bz, by, bx = 16, 16, 32
    nb = (shape[0] // bz) * (shape[1] // by) * (shape[2] // bx)   # 8192 blocks
    seg_ids = rng.integers(0, 2 ** 64, nb, dtype=np.uint64); seg_ids[:50] = 0
    gt_ids = rng.integers(0, 2 ** 32, nb, dtype=np.uint64).astype(np.uint32)
    blk = np.arange(nb).reshape(shape[0] // bz, shape[1] // by, shape[2] // bx)
    full = np.broadcast_to(blk[:, None, :, None, :, None], (shape[0] // bz, bz, shape[1] // by, by, shape[2] // bx, bx)).reshape(shape)
    seg = seg_ids[full]
    gt = gt_ids[(full + (np.arange(shape[1])[None, :, None] >= 256)) % nb]
    m = rng.random(shape) < 0.0015
    seg[m] = rng.integers(0, 2 ** 64, int(m.sum()), dtype=np.uint64)
    s, g = dev(torch, seg), dev(torch, gt)
    ids_s, ids_g, c = s.contingency_table(g)
    os_, og, oc = EV.contingency_triples(seg, gt)
    assert 8 * 10 ** 4 < os_.size < 2 * 10 ** 5
    np.testing.assert_array_equal(ids_s, os_); np.testing.assert_array_equal(ids_g, og); np.testing.assert_array_equal(c, oc)
    st = s.evaluate_statistics(g, (1000,))[0]
    want = EV.statistics(os_, og, oc, 1000)
    for k, v in want.items():
        assert st[k] == (pytest.approx(v, rel=1e-13) if k.startswith("xlog") else v), k
    w = EV.scores(want)
    for k in ("rand_index", "adjusted_rand_index", "fowlkes_mallows_index"):
        assert st[k] == pytest.approx(float(w[k]), rel=1e-12), k
    assert st["variation_of_information"] == pytest.approx(float(w["variation_of_information"]), rel=1e-12)
    assert (st["false_merges"], st["false_splits"]) == w["edit_distance"]


def test_end_to_end_after_connected_components_and_agglomerate(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    rng = np.random.default_rng(7)
    from scipy import ndimage
    prob = ndimage.gaussian_filter(rng.standard_normal((16, 64, 64)), 2.0).astype(np.float32)
    d = DeviceChunk(torch.from_numpy(prob).cuda())
    cc1 = d.connected_component(threshold=0.0)
    cc2 = d.connected_component(threshold=0.05)
    r = cc1.evaluate(cc2)
    w = EV.evaluate(cc1.tensor.cpu().numpy().view(np.uint32), cc2.tensor.cpu().numpy().view(np.uint32))
    for k in ("rand_index", "adjusted_rand_index", "fowlkes_mallows_index"):
        assert same_bits(r[k], w[k]), k
    assert r["variation_of_information"] == pytest.approx(float(w["variation_of_information"]), abs=1e-12)
    assert r["edit_distance"] == w["edit_distance"]
    affs = (1.0 / (1.0 + np.exp(-ndimage.gaussian_filter(rng.standard_normal((3, 16, 48, 48)), (0, 1, 2, 2)) * 20))).astype(np.float32)
    a = DeviceChunk(torch.from_numpy(affs).cuda())
    seg = a.agglomerate(threshold=0.7)
    frag = a.watershed()
    r = seg.evaluate(frag)
    w = EV.evaluate(seg.tensor.cpu().numpy().view(np.uint32), frag.tensor.cpu().numpy().view(np.uint32))
    assert same_bits(r["rand_index"], w["rand_index"]) and r["edit_distance"] == w["edit_distance"]


def test_cli_chain_on_host_chunks(torch):
    from click.testing import CliRunner
    from chunkflow_b200.flow.cli import main
    res = CliRunner().invoke(main, ["create-chunk", "-s", "8", "32", "32", "-p", "sin", "-d", "float32", "-o", "prob",
                                    "connected-components", "-i", "prob", "-o", "chunk", "-t", "0.5",
                                    "connected-components", "-i", "prob", "-o", "groundtruth", "-t", "0.7",
                                    "evaluate-segmentation"], standalone_mode=False)
    assert res.exit_code == 0, (res.output, res.exception)
    task = res.return_value[0]
    from chunkflow_b200.chunk import Chunk
    assert isinstance(task["chunk"], Chunk)
    w = EV.evaluate(task["chunk"].array, task["groundtruth"].array)
    got = task["seg_score"]
    for k in ("rand_index", "adjusted_rand_index", "fowlkes_mallows_index"):
        assert same_bits(got[k], w[k]), k
    assert got["edit_distance"] == w["edit_distance"]
    assert "rand index:" in res.output and "Fowlkes Mallows Index:" in res.output
