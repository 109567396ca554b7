"""`downsample` on the H100 (csrc/downsample.cu through the C ABI, DeviceChunk.downsample and the CLI) against the golden
vectors of the reference's vendored downsampler and the numpy oracle (oracle/downsample_oracle.py), bit for bit."""
import numpy as np
import pytest

from oracle import downsample_oracle as DO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def gold():
    from test_downsample_oracle import GOLDEN
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def to_device(torch, arr, offset=0):
    """A DeviceChunk of ``arr``; ``offset`` elements into a larger buffer, so that the data pointer is not aligned."""
    from chunkflow_b200.chunk.device import DeviceChunk
    arr = np.ascontiguousarray(arr)
    host = arr.view({np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(arr.dtype, arr.dtype))
    flat = torch.from_numpy(np.concatenate([np.zeros(offset, host.dtype), host.ravel()])).cuda()
    return DeviceChunk(flat[offset:].view(arr.shape))


def to_host(d, dtype):
    return d.tensor.cpu().numpy().view(dtype)


def run(torch, arr, factor, offset=0):
    d = to_device(torch, arr, offset)
    before = d.tensor.clone()
    out = d.downsample(factor)
    assert torch.equal(d.tensor, before), "the input was written"
    return to_host(out, arr.dtype)


def test_device_against_golden(torch, gold):
    from test_downsample_oracle import golden_cases
    for name, kind, arr, factor, raises, raises_floor, want in golden_cases(gold):
        a = arr.view(np.uint64) if arr.dtype == np.int64 else arr
        if raises and raises_floor:
            with pytest.raises(ValueError):
                to_device(torch, a).downsample(factor)
            continue
        np.testing.assert_array_equal(run(torch, a, factor).view(want.dtype), want, err_msg=name)


FACTORS = [(2, 2, 2), (1, 2, 2), (2, 1, 2), (2, 2, 1), (4, 4, 4), (1, 4, 4), (3, 3, 1), (2, 4, 4), (3, 2, 5), (1, 1, 1)]


@pytest.mark.parametrize("dtype", [np.uint8, np.uint32, np.uint64, np.int64, np.int32, bool])
@pytest.mark.parametrize("shape", [(8, 16, 34), (7, 33, 65), (6, 31, 100), (16, 64, 96), (7, 33, 64)])
@pytest.mark.parametrize("offset", [0, 1, 3])
def test_every_branch_equals_the_oracle(torch, dtype, shape, offset):
    """Odd and even sizes; int32 / int64 tensors are read as their uint32 / uint64 bit patterns.  uint8 with (1,2,2) and
    (2,2,2) takes the vectorised kernel on rows of a multiple of 16 bytes at offset 0 ((16,64,96), and (7,33,64) with its far
    z and y edges clipped), the generic one on the other shapes and on the views at offsets 1 and 3."""
    rng = np.random.default_rng(shape[2] + offset)
    if dtype == bool:
        arr = rng.random(shape) < 0.5
    elif dtype == np.uint8:
        arr = rng.integers(0, 256, shape, dtype=np.uint8)
    else:
        info = np.iinfo(dtype)
        pool = np.array([0, 1, 2, info.max, info.min, info.max - 1], dtype=dtype)
        arr = pool[rng.integers(0, pool.size, shape)]
        arr[:, :, : shape[2] // 3] = arr[:, :, :1]
    unsigned = {np.dtype(np.int32): np.uint32, np.dtype(np.int64): np.uint64}.get(np.dtype(dtype))
    for f in FACTORS:
        want = DO.downsample(arr.view(unsigned) if unsigned else arr, f)
        got = run(torch, arr, f, offset)
        np.testing.assert_array_equal(got.view(unsigned) if unsigned else got, want, err_msg=f"{dtype} {shape} {f}")


def test_refusals_and_dispatch(torch):
    with pytest.raises(ValueError, match="factor of 0"):
        to_device(torch, np.zeros((8, 8, 8), np.uint32)).downsample((1, 1, 2))
    with pytest.raises(ValueError, match="65793"):
        to_device(torch, np.zeros((8, 8, 8), np.uint8)).downsample((41, 41, 40))
    with pytest.raises(ValueError):
        to_device(torch, np.zeros((8, 8, 8), np.uint8)).downsample((0, 2, 2))
    with pytest.raises(TypeError, match="only support image or segmentation"):
        to_device(torch, np.zeros((8, 8, 8), np.float32)).downsample()
    from chunkflow_b200.chunk.device import DeviceChunk
    with pytest.raises(TypeError, match="only support image or segmentation"):
        DeviceChunk(torch.zeros((2, 4, 4, 4), dtype=torch.uint8, device="cuda")).downsample()


def test_offset_and_voxel_size_bookkeeping(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    d = DeviceChunk(torch.zeros((8, 8, 8), dtype=torch.int64, device="cuda"), voxel_offset=(-3, 5, -8), voxel_size=(40, 4, 4),
                    layer_type="segmentation")
    out = d.downsample((1, 2, 2))
    assert tuple(out.voxel_offset) == (-3, 2, -4) and tuple(out.voxel_size) == (40, 8, 8)
    assert out.layer_type == "segmentation" and out.shape == (8, 4, 4)
    out = d.downsample((3, 2, 5))                                  # strided: ceil(8 / 3) = 3, ceil(8 / 5) = 2
    assert tuple(out.voxel_offset) == (-1, 2, -2) and tuple(out.voxel_size) == (120, 8, 20) and out.shape == (3, 4, 2)
    img = DeviceChunk(torch.zeros((5, 5, 5), dtype=torch.uint8, device="cuda"), voxel_offset=(-1, -1, 7), voxel_size=(1, 1, 1))
    out = img.downsample()
    assert tuple(out.voxel_offset) == (-1, -1, 3) and tuple(out.voxel_size) == (2, 2, 2) and out.shape == (3, 3, 3)


@pytest.mark.parametrize("x", [11373, 11376])
def test_uint8_volume_of_more_than_2_31_voxels(torch, x):
    """Generic kernel (odd rows) and vectorised kernel (rows of a multiple of 16 bytes), odd z and y."""
    from chunkflow_b200.chunk.device import DeviceChunk
    z, y = 17, 11111
    assert z * y * x > 2 ** 31
    a = lambda n, k: torch.arange(n, device="cuda", dtype=torch.int32).view(k)
    t = ((a(z, (z, 1, 1)) * 7 + a(y, (1, y, 1)) * 3 + a(x, (1, 1, x))) % 251).to(torch.uint8)
    out = DeviceChunk(t).downsample((2, 2, 2)).tensor
    ox_last = -(-x // 2) - 1
    assert tuple(out.shape) == (9, 5556, ox_last + 1)
    for oz, oy, ox in ((0, 0, 0), (8, 5555, ox_last), (4, 2000, 4000), (8, 0, ox_last), (3, 5555, 17)):
        block = t[2 * oz: 2 * oz + 2, 2 * oy: 2 * oy + 2, 2 * ox: 2 * ox + 2].cpu().numpy()
        assert int(out[oz, oy, ox]) == int(block.astype(np.int64).sum()) // block.size, (oz, oy, ox)
    del t, out
    torch.cuda.empty_cache()


def test_cli_on_host_and_device_chunks(torch):
    from click.testing import CliRunner
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.flow.cli import main, operator
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (9, 20, 30), dtype=np.uint8)
    seg = np.repeat(rng.integers(0, 5, (9, 20, 15)).astype(np.uint64), 2, axis=2)
    seen = {}

    @main.command("capture-downsample-test")
    @operator
    def capture(tasks):
        for task in tasks:
            seen.update(task)
            yield task
    try:
        @main.command("load-downsample-test")
        @operator
        def load(tasks):
            for task in tasks:
                task["img"] = Chunk(img, voxel_offset=(2, 4, 6), voxel_size=(40, 4, 4))
                task["seg"] = Chunk(seg)
                yield task
        r = CliRunner().invoke(main, ["load-downsample-test", "downsample", "-i", "img", "-o", "mip1",
                                      "downsample", "-i", "mip1", "-o", "mip2", "-f", "1", "2", "2",
                                      "downsample", "-i", "seg", "-o", "seg1",
                                      "to-device", "-i", "seg", "-o", "dseg", "downsample", "-i", "dseg", "-o", "dseg1", "-f", "1", "2", "2",
                                      "capture-downsample-test"], catch_exceptions=False)
        assert r.exit_code == 0, r.output
    finally:
        main.commands.pop("capture-downsample-test", None)
        main.commands.pop("load-downsample-test", None)
    mip1 = DO.downsample(img)
    assert isinstance(seen["mip1"], Chunk) and tuple(seen["mip1"].voxel_offset) == (1, 2, 3)
    assert tuple(seen["mip1"].voxel_size) == (80, 8, 8)
    np.testing.assert_array_equal(seen["mip1"].array, mip1)
    np.testing.assert_array_equal(seen["mip2"].array, DO.downsample(mip1, (1, 2, 2)))
    assert tuple(seen["mip2"].voxel_size) == (80, 16, 16)
    np.testing.assert_array_equal(seen["seg1"].array.view(np.uint64), DO.downsample(seg))
    assert isinstance(seen["dseg1"], DeviceChunk)
    np.testing.assert_array_equal(to_host(seen["dseg1"], np.uint64), DO.downsample(seg, (1, 2, 2)))


def test_thumbnail_chain_against_the_reference(torch, gold):
    """`quantize --mode z` and (1, 2, 2) averagings: the thumbnail pyramid of `save-precomputed --create-thumbnail`, recorded
    from the reference's downsample_and_upload (the last level) and restated by the oracle (every level)."""
    from chunkflow_b200.chunk.device import DeviceChunk
    aff = gold["thumbnail/in"]
    d = DeviceChunk(torch.from_numpy(aff).cuda()).quantize(mode="z")
    for level in DO.thumbnail(aff, int(gold["thumbnail/mip"])):
        d = d.downsample((1, 2, 2))
        np.testing.assert_array_equal(d.tensor.cpu().numpy(), level)
    np.testing.assert_array_equal(d.tensor.cpu().numpy(), gold["thumbnail/out"])
