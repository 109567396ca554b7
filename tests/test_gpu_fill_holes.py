"""`fill-segmentation-holes` on the GPU: DeviceChunk.fill_holes against oracle/fill_holes_oracle.py for every mode and dtype,
counts included, up to 128^3; binary mode against live scipy; the plugin, the command from host and GPU-resident chunks, and
skeletonize(fill_holes=True) against the skeleton of the oracle-filled volume."""
import numpy as np
import pytest
from scipy import ndimage

from oracle import fill_holes_oracle as F
from oracle import skeleton_oracle as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


def nested(shape, seed, n=24):
    """Hollow boxes (some cut by a face) around smaller hollow boxes and single objects, on a background of zeros."""
    rng = np.random.default_rng(seed)
    seg = np.zeros(shape, np.uint32)
    for k in range(1, n + 1):
        size = rng.integers(4, max(5, min(shape) // 2), 3)
        lo = rng.integers(-2, np.maximum(np.array(shape) - size + 2, -1))
        hi = np.minimum(lo + size, shape)
        lo = np.maximum(lo, 0)
        wall = rng.integers(1, 3)
        seg[tuple(slice(a, b) for a, b in zip(lo, hi))] = 13 * k
        seg[tuple(slice(a + wall, b - wall) for a, b in zip(lo, hi))] = 0
        if rng.random() < 0.5:
            c = (lo + hi) // 2
            seg[tuple(slice(a - 1, a + 1) for a in c)] = 13 * k + 5
    return seg


def salt_and_pepper(shape, seed, k=3):
    return np.random.default_rng(seed).integers(0, k, shape).astype(np.uint32)


def typed(seg, dtype):
    if dtype in (np.uint64, np.int64):
        ids = seg.astype(np.uint64)
        ids[ids != 0] += np.uint64(3 << 32)
        return ids.view(np.int64) * -1 if dtype == np.int64 else ids
    if dtype is np.bool_:
        return seg != 0
    if dtype is np.float32:
        return (seg % 7).astype(np.float32) * np.float32(-0.5)   # -0.0 where seg % 7 == 0: background
    return seg.astype(np.int64).astype(dtype)


def device_chunk(torch, arr, **kw):
    from chunkflow_b200.chunk.device import DeviceChunk
    arr = np.ascontiguousarray(arr)
    host = arr.view({4: np.int32, 8: np.int64}[arr.itemsize]) if arr.dtype in (np.uint32, np.uint64) else arr
    return DeviceChunk(torch.from_numpy(host).cuda(), **kw)


def host_of(dev, dtype):
    return dev.tensor.cpu().numpy().view(dtype)


CASES = [("nested", (64, 64, 64)), ("nested", (128, 128, 128)), ("salt_and_pepper", (20, 30, 40)), ("nested", (1, 96, 80)),
         ("nested", (33, 17, 129))]


@pytest.mark.parametrize("mode", F.MODES)
@pytest.mark.parametrize("name, shape", CASES)
def test_fill_holes_equals_the_oracle(torch, name, shape, mode):
    seg = nested(shape, shape[0]) if name == "nested" else salt_and_pepper(shape, 1)
    dtypes = F.BINARY_DTYPES if mode == "binary" else F.OBJECT_DTYPES
    for dtype in dtypes:
        arr = typed(seg, dtype)
        want, n = F.fill(arr, mode)
        st = {}
        got, m = device_chunk(torch, arr).fill_holes(mode, return_fill_count=True, stats=st)
        got = host_of(got, arr.dtype)
        assert got.dtype == arr.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)) and m == n, (dtype, m, n, st)
    if name == "nested" and min(shape) > 1:
        assert n > 0


def test_binary_is_live_scipy(torch):
    rng = np.random.default_rng(7)
    for p in (0.3, 0.5, 0.7):
        arr = (rng.random((96, 100, 104)) < p).astype(np.uint8)
        got, m = device_chunk(torch, arr).fill_holes(return_fill_count=True)
        want = ndimage.binary_fill_holes(arr)
        assert np.array_equal(host_of(got, np.uint8), want.astype(np.uint8)) and m == int((want & (arr == 0)).sum())


def test_all_zero_single_id_and_refusals(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    for arr in (np.zeros((5, 6, 7), np.uint32), np.full((5, 6, 7), 9, np.uint32)):
        for mode in F.MODES:
            got, m = device_chunk(torch, arr).fill_holes(mode, return_fill_count=True)
            assert np.array_equal(host_of(got, np.uint32), F.fill(arr, mode)[0]) and m == 0
    with pytest.raises(TypeError, match="keep-enclosed mode takes"):
        DeviceChunk(torch.zeros((4, 4, 4), dtype=torch.uint8, device="cuda")).fill_holes("keep-enclosed")
    with pytest.raises(TypeError, match="binary mode takes"):
        DeviceChunk(torch.zeros((4, 4, 4), dtype=torch.float64, device="cuda")).fill_holes()
    with pytest.raises(ValueError, match="mode"):
        DeviceChunk(torch.zeros((4, 4, 4), dtype=torch.int32, device="cuda")).fill_holes("holes")
    with pytest.raises(ValueError):
        DeviceChunk(torch.zeros((1, 4, 4, 4), dtype=torch.int32, device="cuda")).fill_holes()


def test_segmentation_fill_holes_on_a_host_chunk(torch):
    from chunkflow_b200.chunk.segmentation import Segmentation
    seg = nested((40, 48, 56), 3)
    s = Segmentation(seg, voxel_offset=(1, 2, 3), voxel_size=(40, 4, 4))
    out, n = s.fill_holes("keep-enclosed", return_fill_count=True)
    want, m = F.fill(seg, "keep-enclosed")
    assert isinstance(out, Segmentation) and np.array_equal(out.array, want) and n == m and tuple(out.voxel_offset) == (1, 2, 3)


def test_plugin_returns_a_chunk_with_the_properties(torch):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.plugins import fill_segmentation_holes as plugin
    seg = nested((32, 40, 48), 5)
    for chunk in (Chunk(seg, voxel_offset=(3, 4, 5), voxel_size=(40, 4, 4), layer_type="segmentation"),
                  device_chunk(torch, seg, voxel_offset=(3, 4, 5), voxel_size=(40, 4, 4), layer_type="segmentation")):
        out = plugin.execute(chunk)
        assert isinstance(out, list) and len(out) == 1 and isinstance(out[0], Chunk)
        dtype = np.uint32 if isinstance(chunk, Chunk) else np.int32   # a DeviceChunk holds uint32 ids as int32
        assert out[0].array.dtype == dtype and np.array_equal(out[0].array.view(np.uint32), F.fill(seg, "binary")[0])
        assert tuple(out[0].voxel_offset) == (3, 4, 5) and tuple(out[0].voxel_size) == (40, 4, 4)
        assert out[0].layer_type == "segmentation"


@pytest.mark.parametrize("to_device", [False, True])
@pytest.mark.parametrize("mode", F.MODES)
def test_command_from_host_and_gpu_resident_chunks(torch, to_device, mode):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.flow.cli import main
    seg = nested((24, 40, 48), 9)
    chunk = Chunk(seg, voxel_offset=(1, 2, 3), voxel_size=(40, 4, 4))
    if to_device:
        chunk = device_chunk(torch, seg, voxel_offset=(1, 2, 3), voxel_size=(40, 4, 4))
    op = main.commands["fill-segmentation-holes"].callback(input_chunk_name="chunk", output_chunk_name="filled", mode=mode)
    task = list(op(iter([{"log": {"timer": {}}, "chunk": chunk}])))[0]
    out = task["filled"]
    assert isinstance(out, DeviceChunk) == to_device
    arr = host_of(out, np.uint32) if to_device else out.array
    assert np.array_equal(arr, F.fill(seg, mode)[0]) and tuple(out.voxel_offset) == (1, 2, 3)
    assert main.commands["fill-segmentation-holes"].help.startswith("(extension)")


def test_skeletonize_after_filling_is_the_skeleton_of_the_filled_volume(torch):
    from chunkflow_b200.flow.cli import main
    seg = nested((24, 48, 56), 11, 10)
    filled, n = F.fill(seg, "remove-enclosed")
    assert n > 0
    p = dict(voxel_size=(40, 4, 4), const=40, scale=2, dust_threshold=5)
    got = device_chunk(torch, seg).skeletonize(fill_holes=True, **p)
    want = S.skeletonize(filled, p["voxel_size"], const=40, scale=2, dust_threshold=5)
    assert list(got) == list(want)
    for k, (v, e, r) in want.items():
        assert np.array_equal(got[k].vertices, v) and np.array_equal(got[k].edges, e) and np.array_equal(got[k].radii, r), k
    assert any(o.name == "fill_holes" for o in main.commands["skeletonize"].params)
