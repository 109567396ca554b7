"""Segmentation clean-up on the H100 (csrc/relabel.cu through the C ABI, DeviceChunk.unique / mask_fragments / mask_except /
remap, the host Segmentation methods and the CLI) against the golden vectors of the real reference's methods and the numpy
oracle (oracle/relabel_oracle.py)."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

from oracle import evaluation_oracle as EV
from oracle import relabel_oracle as RO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def gold():
    from test_relabel_oracle import GOLDEN
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def dev(arr):
    from chunkflow_b200.chunk.segmentation import _device_labels
    return _device_labels(np.asarray(arr), "cuda:0")


def host(d, dtype=None):
    """The labels of a DeviceChunk as unsigned numpy values."""
    a = d.tensor.cpu().numpy()
    a = a.view({np.dtype(np.int32): np.uint32, np.dtype(np.int64): np.uint64}.get(a.dtype, a.dtype))
    return a if dtype is None else a.astype(dtype)


def labels(rng, shape, dtype, pool_size=60, runs=True):
    """Random ids (0, 2^63 + 5 and 2^64 - 1 among the uint64 ones), half of every row one long run when ``runs``."""
    if dtype == np.uint64:
        pool = np.unique(np.concatenate([np.array([0, 2 ** 63 + 5, 2 ** 64 - 1, 1], np.uint64),
                                         rng.integers(0, 2 ** 64, pool_size, dtype=np.uint64)]))
    else:
        pool = np.unique(np.concatenate([[0, 1], rng.integers(0, np.iinfo(dtype).max, pool_size, endpoint=True)])).astype(dtype)
    a = pool[rng.integers(0, pool.size, shape)]
    if runs:
        a[:, :, : shape[2] // 2] = a[:, :, :1]
    return a


def test_device_against_golden(torch, gold):
    from test_relabel_oracle import golden_calls
    for name, arr, method, arg, want, ret, _ in golden_calls(gold):
        d = dev(arr)
        if method == "remap":
            assert d.remap(arg) == ret, (name, arg)
            assert d.tensor.dtype == torch.int64
        elif method == "mask_fragments":
            num, masked = d.mask_fragments(arg)
            ids, counts = np.unique(arr, return_counts=True)
            assert (num, masked) == (ids.size, int((counts <= arg).sum()))
        else:
            d.mask_except(arg)
        np.testing.assert_array_equal(host(d, want.dtype), want, err_msg=f"{name} {method} {arg}")


@pytest.mark.parametrize("dtype", [np.uint8, np.uint32, np.uint64])
@pytest.mark.parametrize("shape", [(3, 5, 7), (4, 33, 65), (2, 31, 1000), (16, 64, 96)])
def test_unique_masks_and_remap_equal_the_oracle(torch, dtype, shape):
    """Sizes that are no multiple of the vector width or of a warp's 32 loads; long runs next to salt and pepper."""
    rng = np.random.default_rng(shape[2])
    arr = labels(rng, shape, dtype)
    ids, counts = dev(arr).unique(return_counts=True)
    o_ids, o_counts = RO.unique(arr, return_counts=True)
    assert ids.dtype == arr.dtype
    np.testing.assert_array_equal(ids, o_ids); np.testing.assert_array_equal(counts, o_counts)
    np.testing.assert_array_equal(dev(arr).unique(), o_ids)
    thr = int(np.sort(o_counts)[o_counts.size // 2])          # some count equals the threshold
    d = dev(arr)
    before = d.tensor.data_ptr()
    assert d.mask_fragments(thr) == (o_ids.size, int((o_counts <= thr).sum()))
    assert d.tensor.data_ptr() == before and d.tensor.shape == arr.shape   # in place
    np.testing.assert_array_equal(host(d), RO.mask_fragments(arr, thr)[0])
    keep = [int(i) for i in o_ids[::3]] + [12345]
    d = dev(arr)
    d.mask_except(keep)
    np.testing.assert_array_equal(host(d), RO.mask_except_ids(arr, keep))
    d = dev(arr)
    d.mask_except([])
    assert not host(d).any()
    d = dev(arr)
    want, new_max = RO.remap(arr, 7)
    assert d.remap(7) == new_max
    np.testing.assert_array_equal(host(d), want)


def test_salt_and_pepper_and_one_long_run(torch):
    rng = np.random.default_rng(1)
    salt = labels(rng, (8, 64, 64), np.uint64, pool_size=3000, runs=False)
    d = dev(salt)
    want, new_max = RO.remap(salt, 0)
    assert d.remap() == new_max
    np.testing.assert_array_equal(host(d), want)
    one = np.full((5, 40, 50), 2 ** 64 - 1, np.uint64)
    one[2, 20, 25:] = 3
    d = dev(one)
    assert d.remap(10) == 12
    np.testing.assert_array_equal(host(d), RO.remap(one, 10)[0])


def test_table_grows_from_a_small_start(torch):
    from chunkflow_b200 import _native
    rng = np.random.default_rng(5)
    arr = labels(rng, (8, 32, 32), np.uint64, pool_size=500, runs=False)
    d = dev(arr)
    work = torch.empty(_native.label_table_workspace(arr.size, 32), dtype=torch.uint8, device="cuda:0")
    with pytest.raises(_native.NativeError) as err:
        _native.label_table_device(d.tensor.data_ptr(), _native.DTYPE_U64, arr.shape, work.data_ptr(), 32)
    assert err.value.code == _native.ERR_CAPACITY
    with pytest.raises(_native.NativeError) as err:    # an incomplete table is not applied
        _native.label_apply_device(d.tensor.data_ptr(), _native.DTYPE_U64, arr.size, work.data_ptr(), 32, d.tensor.data_ptr(),
                                   _native.DTYPE_U64)
    assert err.value.code == _native.ERR_INVALID_ARGUMENT
    ids, counts = d.unique(return_counts=True, table_slots=32)
    o_ids, o_counts = RO.unique(arr, return_counts=True)
    np.testing.assert_array_equal(ids, o_ids); np.testing.assert_array_equal(counts, o_counts)
    want, new_max = RO.remap(arr, 0)
    assert d.remap(table_slots=32) == new_max
    np.testing.assert_array_equal(host(d), want)


def test_remap_refuses_bad_base_ids(torch):
    from chunkflow_b200 import _native
    arr = np.arange(24, dtype=np.uint32).reshape(2, 3, 4)
    with pytest.raises(ValueError):
        dev(arr).remap(-1)
    d = dev(arr)
    with pytest.raises(_native.NativeError) as err:    # 23 labels + base id > 2^64 - 1
        d.remap(2 ** 64 - 23)
    assert err.value.code == _native.ERR_INVALID_ARGUMENT
    np.testing.assert_array_equal(host(d), arr)         # untouched
    assert dev(arr).remap(2 ** 64 - 24) == 2 ** 64 - 1


def test_dust_and_keep_list_in_one_call_equal_the_two_calls(torch, capsys):
    from chunkflow_b200.chunk.segmentation import mask_out_objects
    rng = np.random.default_rng(8)
    arr = labels(rng, (6, 40, 70), np.uint32, pool_size=200)
    ids, counts = np.unique(arr, return_counts=True)
    keep = set(int(i) for i in ids[::2])
    one = dev(arr)
    mask_out_objects(one, 30, keep)
    two = dev(arr)
    two.mask_fragments(30)
    two.mask_except(keep)
    want, text = RO.mask_out_objects(arr, 30, keep)
    np.testing.assert_array_equal(host(one), want); np.testing.assert_array_equal(host(two), want)
    assert capsys.readouterr().out == text


def test_remap_is_idempotent_and_chained_base_ids_are_disjoint(torch):
    rng = np.random.default_rng(9)
    a, b = labels(rng, (4, 30, 50), np.uint32), labels(rng, (4, 30, 50), np.uint64)
    da, db = dev(a), dev(b)
    base = da.remap()
    first = host(da).copy()
    assert da.remap() == base
    np.testing.assert_array_equal(host(da), first)
    top = db.remap(base)
    ia, ib = np.unique(first[first != 0]), np.unique(host(db)[host(db) != 0])
    assert ia.size == base and ib.min() == base + 1 and ib.max() == top == base + ib.size
    assert not np.intersect1d(ia, ib).size


def test_evaluate_of_a_remapped_segmentation_is_bitwise_equal(torch):
    rng = np.random.default_rng(10)
    seg, gt = labels(rng, (8, 48, 64), np.uint64, pool_size=150), labels(rng, (8, 48, 64), np.uint32, pool_size=90)
    base = dev(seg).evaluate_statistics(dev(gt), (0, 10, 1000))
    d = dev(seg)
    d.remap(2 ** 40)
    again = d.evaluate_statistics(dev(gt), (0, 10, 1000))
    for x, y in zip(base, again):
        for k in ("rand_index", "adjusted_rand_index", "variation_of_information", "fowlkes_mallows_index", "false_merges",
                  "false_splits"):
            assert np.float64(x[k]).tobytes() == np.float64(y[k]).tobytes(), k


def test_segmentation_host_methods_print_and_return_like_the_golden(torch, gold):
    from chunkflow_b200.chunk.segmentation import Segmentation
    from test_relabel_oracle import golden_calls
    for name, arr, method, arg, want, ret, printed in golden_calls(gold):
        seg = Segmentation(arr.copy())
        buf = io.StringIO()
        with redirect_stdout(buf):
            r = getattr(seg, method)(arg)
        assert seg.array.dtype == want.dtype, (name, method)
        np.testing.assert_array_equal(seg.array, want, err_msg=f"{name} {method} {arg}")
        assert buf.getvalue() == printed, (name, method, arg)
        assert (r is None and ret is None) or (isinstance(r, np.uint64) and int(r) == ret)


def test_cli_chain_stays_on_the_device(torch, monkeypatch):
    from click.testing import CliRunner
    from scipy import ndimage
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.flow import cli
    rng = np.random.default_rng(12)
    affs = (1.0 / (1.0 + np.exp(-ndimage.gaussian_filter(rng.standard_normal((3, 16, 48, 48)), (0, 1, 2, 2)) * 20))).astype(np.float32)
    gt = labels(rng, (16, 48, 48), np.uint32, pool_size=20)
    seen = {}

    @cli.main.command("probe")
    @cli.operator
    def probe(tasks):
        for task in tasks:
            task["affs"], task["groundtruth"] = Chunk(affs), Chunk(gt)
            yield task

    @cli.main.command("peek")
    @cli.operator
    def peek(tasks):
        for task in tasks:
            assert isinstance(task["chunk"], DeviceChunk)
            seen[len(seen)] = host(task["chunk"]).copy()
            yield task

    downloads = []
    to_chunk = DeviceChunk.to_chunk
    monkeypatch.setattr(DeviceChunk, "to_chunk", lambda self: downloads.append(1) or to_chunk(self))
    try:
        res = CliRunner().invoke(cli.main, ["probe", "to-device", "-i", "affs", "-o", "chunk", "agglomerate", "peek",
                                            "mask-out-objects", "-d", "100", "peek", "remap-segmentation", "peek",
                                            "evaluate-segmentation", "to-host"], standalone_mode=False)
    finally:
        cli.main.commands.pop("probe"); cli.main.commands.pop("peek")
    assert res.exit_code == 0, (res.output, res.exception)
    task = res.return_value[0]
    assert len(downloads) == 1 and isinstance(task["chunk"], Chunk)      # only `to-host` brought voxels back
    agg, masked, remapped = seen[0], seen[1], seen[2]
    want_masked, line = RO.mask_fragments(agg, 100)
    np.testing.assert_array_equal(masked, want_masked)
    assert line in res.output
    want, new_max = RO.remap(want_masked, 0)
    np.testing.assert_array_equal(remapped, want)
    np.testing.assert_array_equal(task["chunk"].array.view(np.uint64), want)
    assert task["base_id"] == new_max
    w = EV.evaluate(want, gt)
    for k in ("rand_index", "adjusted_rand_index", "fowlkes_mallows_index"):
        assert np.float64(task["seg_score"][k]).tobytes() == np.float64(w[k]).tobytes(), k
    assert task["seg_score"]["edit_distance"] == w["edit_distance"]


def test_cli_on_host_chunks_and_chained_base_id(torch):
    from click.testing import CliRunner
    from chunkflow_b200.chunk.segmentation import Segmentation
    from chunkflow_b200.flow.cli import main
    res = CliRunner().invoke(main, ["create-chunk", "-s", "8", "32", "32", "-p", "sin", "-d", "float32", "-o", "prob",
                                    "connected-components", "-i", "prob", "-o", "a", "-t", "0.5",
                                    "connected-components", "-i", "prob", "-o", "b", "-t", "0.7",
                                    "mask-out-objects", "-i", "a", "-o", "a", "-d", "3", "-s", "1,2,3",
                                    "remap-segmentation", "-i", "a", "-o", "a", "--base-id", "100",
                                    "remap-segmentation", "-i", "b", "-o", "b"], standalone_mode=False)
    assert res.exit_code == 0, (res.output, res.exception)
    task = res.return_value[0]
    a, b = task["a"], task["b"]
    assert isinstance(a, Segmentation) and isinstance(b, Segmentation) and a.array.dtype == b.array.dtype == np.uint64
    ia, ib = np.unique(a.array[a.array != 0]), np.unique(b.array[b.array != 0])
    assert ia.min() == 101 and ib.min() == ia.max() + 1 and task["base_id"] == ib.max()
    assert "masking out" in res.output
