"""`gaussian-filter` and the median filter on the H100 (csrc/filters.cu through the C ABI, DeviceChunk, Chunk, the CLI and the
two plugins) against live scipy.ndimage and the golden vectors of the reference's own callers, bit for bit."""
import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import filters_oracle as FO

pytestmark = pytest.mark.gpu
MODES = tuple(FO.MODES)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def gold():
    from test_filters_oracle import GOLDEN
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def to_device(torch, arr, offset=0, **kw):
    """A DeviceChunk of ``arr``; ``offset`` elements into a larger buffer, so that the data pointer is not aligned."""
    from chunkflow_b200.chunk.device import DeviceChunk
    arr = np.ascontiguousarray(arr)
    flat = torch.from_numpy(np.concatenate([np.zeros(offset, arr.dtype), arr.ravel()])).cuda()
    return DeviceChunk(flat[offset:].view(arr.shape), **kw)


def gaussian(torch, arr, sigma, offset=0, per_channel=False):
    d = to_device(torch, arr, offset)
    d.gaussian_filter_2d(sigma, per_channel=per_channel)
    return d.tensor.cpu().numpy()


def median(torch, arr, size, mode, offset=0):
    d = to_device(torch, arr, offset)
    before = d.tensor.clone()
    out = d.median_filter(size, mode)
    assert torch.equal(d.tensor, before), "the input was written"
    return out.tensor.cpu().numpy()


def scipy_sections(arr, sigma):
    """The reference's method: gaussian_filter of every [..., z, :, :]."""
    out = arr.copy()
    for z in range(arr.shape[-3]):
        out[..., z, :, :] = ndi.gaussian_filter(arr[..., z, :, :], sigma)
    return out


def test_device_against_golden(torch, gold):
    from test_filters_oracle import golden_cases
    for name, caller, arr, kw, want in golden_cases(gold):
        if caller == "median_plugin":
            got = median(torch, arr, kw["size"], kw["mode"])
        else:
            got = gaussian(torch, arr, kw["sigma"], per_channel=caller == "gaussian_plugin")
        assert got.dtype == want.dtype
        np.testing.assert_array_equal(got, want, err_msg=name)


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("shape", [(3, 100, 300), (2, 257, 129), (2, 31, 1000), (1, 2, 500), (3, 700, 1)])
@pytest.mark.parametrize("offset", [0, 1, 3])
def test_gaussian_equals_scipy(torch, dtype, shape, offset):
    rng = np.random.default_rng(sum(shape) + offset)
    a = rng.integers(0, 256, shape, dtype=np.uint8) if dtype == np.uint8 else (rng.random(shape) * 100).astype(np.float32)
    for s in (0.5, 1, 2, 3.7, (0, 1), (1, 2), 16):
        np.testing.assert_array_equal(gaussian(torch, a, s, offset), scipy_sections(a, s), err_msg=str(s))


@pytest.mark.parametrize("channels", [3, 4])
def test_gaussian_on_affinity_maps(torch, channels):
    """The command runs across the channels (the reference's quirk), the plugin channel by channel."""
    a = np.random.default_rng(channels).random((channels, 9, 130, 150), dtype=np.float32)
    for s in (1, 2, (1, 0.5, 2), (0, 1, 1)):
        np.testing.assert_array_equal(gaussian(torch, a, s, offset=1), scipy_sections(a, s), err_msg=str(s))
    per_channel = np.stack([scipy_sections(a[c], 1.5) for c in range(channels)])
    np.testing.assert_array_equal(gaussian(torch, a, 1.5, per_channel=True), per_channel)


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("offset", [0, 1])
def test_median_equals_scipy(torch, dtype, offset):
    rng = np.random.default_rng(7 + offset)
    for shape in ((40, 70, 90), (1, 2, 33), (2, 1, 5), (5, 33, 2)):
        a = rng.integers(0, 7, shape).astype(dtype) if dtype == np.uint8 else rng.random(shape).astype(np.float32)
        for mode in MODES:
            for size in ((3, 1, 1), (1, 3, 3), (3, 3, 3), (2, 2, 2), (5, 5, 5), (4, 1, 2), (5, 1, 1), 1):
                np.testing.assert_array_equal(median(torch, a, size, mode, offset), ndi.median_filter(a, size=size, mode=mode),
                                              err_msg=f"{shape} {mode} {size}")
    aff = rng.random((3, 6, 20, 30)).astype(dtype)
    for size in ((1, 3, 1, 1), (3, 3, 1, 1), 2):
        np.testing.assert_array_equal(median(torch, aff, size, "reflect", offset), ndi.median_filter(aff, size=size))


def test_refusals(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    d = to_device(torch, np.zeros((4, 8, 8), np.uint8))
    with pytest.raises(ValueError, match="64"):
        d.gaussian_filter_2d(16.2)
    with pytest.raises(RuntimeError, match="sequence argument"):
        d.gaussian_filter_2d((1, 1, 1))
    with pytest.raises(ValueError, match="125"):
        d.median_filter((6, 5, 5))
    with pytest.raises(RuntimeError, match="sequence argument"):
        d.median_filter((3, 1))
    with pytest.raises(RuntimeError, match="sequence argument"):
        to_device(torch, np.zeros((3, 4, 8, 8), np.float32)).median_filter((3, 1, 1))
    with pytest.raises(RuntimeError, match="boundary mode"):
        d.median_filter(3, "edge")
    for dt in (torch.int32, torch.float64, torch.int16):
        bad = DeviceChunk(torch.zeros((4, 8, 8), dtype=dt, device="cuda"))
        with pytest.raises(TypeError):
            bad.gaussian_filter_2d(1)
        with pytest.raises(TypeError):
            bad.median_filter()


def test_uint8_chunk_of_more_than_2_31_voxels(torch):
    """64-bit indexing: the median's z walk, then the gaussian in place, checked on the first, a middle and the last section."""
    from chunkflow_b200.chunk.device import DeviceChunk
    z, y, x = 17, 11111, 11373
    assert z * y * x > 2 ** 31
    a = lambda n, k: torch.arange(n, device="cuda", dtype=torch.int32).view(k)
    t = ((a(z, (z, 1, 1)) * 7 + a(y, (1, y, 1)) * 13 + a(x, (1, 1, x)) * 5) % 251).to(torch.uint8)
    d = DeviceChunk(t)
    med = d.median_filter((3, 1, 1)).tensor
    for k in (0, 8, z - 1):
        lo, hi = max(k - 1, 0), min(k + 1, z - 1)        # reflect: z -1 -> 0, z -> z - 1
        want = np.median(np.stack([t[lo].cpu().numpy(), t[k].cpu().numpy(), t[hi].cpu().numpy()]), axis=0).astype(np.uint8)
        np.testing.assert_array_equal(med[k].cpu().numpy(), want, err_msg=str(k))
    del med
    sections = {k: t[k].cpu().numpy() for k in (0, 8, z - 1)}
    d.gaussian_filter_2d(1)
    for k, sec in sections.items():
        np.testing.assert_array_equal(t[k].cpu().numpy(), ndi.gaussian_filter(sec, 1), err_msg=str(k))
    del t, d
    torch.cuda.empty_cache()


def test_host_chunk_method_writes_back_in_place(torch):
    from chunkflow_b200.chunk import Chunk
    arr = np.random.default_rng(3).random((3, 4, 40, 50), dtype=np.float32)
    want = scipy_sections(arr, 2)
    view = arr[1]
    c = Chunk(arr, voxel_offset=(1, 2, 3))
    assert c.gaussian_filter_2d(2) is None
    assert c.array is arr
    np.testing.assert_array_equal(arr, want)
    np.testing.assert_array_equal(view, want[1])


def test_cli_chains_on_host_and_device_chunks(torch):
    from click.testing import CliRunner
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.flow.cli import main, operator
    img = np.random.default_rng(5).integers(0, 256, (9, 40, 60), dtype=np.uint8)
    host = img.copy()
    view = host[4]
    seen = {}

    @main.command("capture-filters-test")
    @operator
    def capture(tasks):
        for task in tasks:
            seen.update(task)
            yield task
    try:
        @main.command("load-filters-test")
        @operator
        def load(tasks):
            for task in tasks:
                task["img"] = Chunk(host, voxel_offset=(2, 4, 6), voxel_size=(40, 4, 4))
                task["dimg"] = Chunk(img.copy(), voxel_offset=(2, 4, 6), voxel_size=(40, 4, 4))
                yield task
        r = CliRunner().invoke(main, ["load-filters-test",
                                      "gaussian-filter", "-i", "img", "-s", "1", "median-filter", "-i", "img", "-o", "med",
                                      "to-device", "-i", "dimg", "-o", "dimg", "gaussian-filter", "-i", "dimg", "-s", "1",
                                      "median-filter", "-i", "dimg", "-o", "dmed", "--mode", "nearest", "--size", "1", "3", "3",
                                      "to-host", "-i", "dmed", "-o", "hmed", "capture-filters-test"], catch_exceptions=False)
        assert r.exit_code == 0, r.output
        r = CliRunner().invoke(main, ["create-chunk", "-s", "8", "30", "40", "-d", "float32", "-t", "1", "2", "3", "-e", "4", "5", "6",
                                      "to-device", "gaussian-filter", "-s", "1", "median-filter", "to-host",
                                      "capture-filters-test"], catch_exceptions=False)
        assert r.exit_code == 0, r.output
    finally:
        main.commands.pop("capture-filters-test", None)
        main.commands.pop("load-filters-test", None)
    blurred = scipy_sections(img, 1)
    np.testing.assert_array_equal(host, blurred)            # written in place into the task's array
    np.testing.assert_array_equal(view, blurred[4])
    assert isinstance(seen["med"], Chunk) and tuple(seen["med"].voxel_offset) == (2, 4, 6)
    assert tuple(seen["med"].voxel_size) == (40, 4, 4)
    np.testing.assert_array_equal(seen["med"].array, ndi.median_filter(blurred, size=(3, 1, 1)))
    assert isinstance(seen["dimg"], DeviceChunk) and isinstance(seen["dmed"], DeviceChunk)
    np.testing.assert_array_equal(seen["dimg"].tensor.cpu().numpy(), blurred)
    assert tuple(seen["dmed"].voxel_offset) == (2, 4, 6)
    np.testing.assert_array_equal(seen["hmed"].array, ndi.median_filter(blurred, size=(1, 3, 3), mode="nearest"))
    assert tuple(seen["hmed"].voxel_size) == (40, 4, 4)
    created = Chunk.create(size=(8, 30, 40), dtype=np.float32).array
    np.testing.assert_array_equal(seen["chunk"].array, ndi.median_filter(scipy_sections(created, 1), size=(3, 1, 1)))
    assert tuple(seen["chunk"].voxel_offset) == (1, 2, 3) and tuple(seen["chunk"].voxel_size) == (4, 5, 6)


def test_plugins_with_host_and_device_chunks(torch):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.plugins import gaussian_filter, median_filter
    aff = np.random.default_rng(9).random((3, 5, 30, 40), dtype=np.float32)
    per_channel = np.stack([scipy_sections(aff[c], 1) for c in range(3)])
    c = Chunk(aff.copy(), voxel_offset=(1, 2, 3), voxel_size=(4, 4, 40))
    out = gaussian_filter.execute(c)
    assert out is not c and np.array_equal(c.array, aff) and tuple(out.voxel_offset) == (1, 2, 3)
    np.testing.assert_array_equal(out.array, per_channel)
    assert gaussian_filter.execute(c, sigma=1, inplace=True) is c
    np.testing.assert_array_equal(c.array, per_channel)
    d = to_device(torch, aff, voxel_offset=(1, 2, 3))
    out = gaussian_filter.execute(d, sigma=1)
    assert isinstance(out, DeviceChunk) and out is not d and np.array_equal(d.tensor.cpu().numpy(), aff)
    np.testing.assert_array_equal(out.tensor.cpu().numpy(), per_channel)
    assert gaussian_filter.execute(d, sigma=1, inplace=True) is d
    np.testing.assert_array_equal(d.tensor.cpu().numpy(), per_channel)

    img = np.random.default_rng(10).integers(0, 256, (9, 30, 40), dtype=np.uint8)
    res = median_filter.execute(Chunk(img))
    assert isinstance(res, list) and len(res) == 1 and isinstance(res[0], np.ndarray)
    np.testing.assert_array_equal(res[0], ndi.median_filter(img, size=(3, 1, 1), mode="reflect"))
    res = median_filter.execute(to_device(torch, img, voxel_offset=(5, 5, 5)), size=(1, 3, 3), mode="mirror")
    assert isinstance(res[0], DeviceChunk) and tuple(res[0].voxel_offset) == (5, 5, 5)
    np.testing.assert_array_equal(res[0].tensor.cpu().numpy(), ndi.median_filter(img, size=(1, 3, 3), mode="mirror"))
