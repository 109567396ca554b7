"""`clahe` on the H100 (csrc/clahe.cu through the C ABI, DeviceChunk, the plugin and the CLI) against the golden vectors of the
reference's own plugin and, where OpenCV is importable, against live cv2, bit for bit."""
import numpy as np
import pytest

from oracle import clahe_oracle as CO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def gold():
    from test_clahe_oracle import GOLDEN
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def to_device(torch, arr, offset=0, **kw):
    """A DeviceChunk of ``arr``; ``offset`` bytes into a larger buffer, so that the data pointer is not aligned."""
    from chunkflow_b200.chunk.device import DeviceChunk
    arr = np.ascontiguousarray(arr)
    flat = torch.from_numpy(np.concatenate([np.zeros(offset, arr.dtype), arr.ravel()])).cuda()
    return DeviceChunk(flat[offset:].view(arr.shape), **kw)


def clahe(torch, arr, clip, grid, offset=0):
    d = to_device(torch, arr, offset)
    before = d.tensor.clone()
    out = d.clahe(clip, grid)
    assert torch.equal(d.tensor, before), "the input was written"
    assert out.tensor.data_ptr() != d.tensor.data_ptr()
    return out.tensor.cpu().numpy()


def cv2_sections(arr, clip, grid):
    cv2 = pytest.importorskip("cv2")
    c = cv2.createCLAHE(clip, tuple(grid))
    return np.stack([c.apply(s) for s in arr])


def test_device_against_golden(torch, gold):
    from test_clahe_oracle import golden_cases
    for name, a, clip, grid, want in golden_cases(gold):
        for offset in (0, 7):
            np.testing.assert_array_equal(clahe(torch, a, clip, grid, offset), want, err_msg=f"{name} {offset}")


@pytest.mark.parametrize("offset", [0, 1, 3, 8, 15])
def test_equals_cv2_on_unaligned_views_and_odd_rows(torch, offset):
    rng = np.random.default_rng(offset)
    for shape in ((3, 100, 333), (2, 257, 129), (4, 31, 1000), (2, 1, 517), (3, 300, 1)):
        a = rng.integers(0, 256, shape, dtype=np.uint8)
        for grid, clip in (((8, 8), 2.0), ((18, 26), 5.0), ((512, 512), 20.0), ((3, 7), 0.0), ((64, 2), 40.0)):
            np.testing.assert_array_equal(clahe(torch, a, clip, grid, offset), cv2_sections(a, clip, grid),
                                          err_msg=f"{shape} {grid} {clip}")


def test_both_paths_and_the_threshold_edge(torch):
    """Tile sizes from 1 pixel to whole sections, through the last small-tile size and the first table size."""
    from test_clahe_oracle import SMALL_TILE_MAX, tile_pixels
    rng = np.random.default_rng(1)
    sizes = set()
    for y, x in ((128, 128), (130, 127), (96, 200)):
        a = rng.integers(0, 256, (3, y, x), dtype=np.uint8)
        for grid in ((128, 128), (64, 64), (32, 64), (32, 32), (16, 32), (16, 16), (8, 8), (40, 9), (1, 1)):
            sizes.add(tile_pixels(y, x, grid))
            np.testing.assert_array_equal(clahe(torch, a, 3.0, grid), CO.clahe(a, 3.0, grid), err_msg=f"{y} {x} {grid}")
    assert min(sizes) == 1 and SMALL_TILE_MAX in sizes and any(SMALL_TILE_MAX < t <= 2 * SMALL_TILE_MAX for t in sizes)


def test_workspace_batches(torch):
    """A (64, 32) grid on 512^2 sections: 128-pixel tiles, 512 KiB of LUTs per section, so 70 sections run in two batches."""
    from chunkflow_b200 import _native
    assert _native.clahe_workspace((70, 512, 512), (64, 32)) == 64 * 2048 * 256
    a = np.random.default_rng(2).integers(0, 256, (70, 512, 512), dtype=np.uint8)
    got = clahe(torch, a, 2.0, (64, 32))
    for k in (0, 63, 64, 69):
        np.testing.assert_array_equal(got[k], CO.apply_section(a[k], 2.0, (64, 32)), err_msg=str(k))


def test_refusals(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    for dt in (torch.uint16 if hasattr(torch, "uint16") else torch.int16, torch.float32, torch.int32):
        with pytest.raises(TypeError):
            DeviceChunk(torch.zeros((4, 8, 8), dtype=dt, device="cuda")).clahe()
    with pytest.raises(ValueError):
        DeviceChunk(torch.zeros((2, 4, 8, 8), dtype=torch.uint8, device="cuda")).clahe()
    d = DeviceChunk(torch.zeros((4, 8, 8), dtype=torch.uint8, device="cuda"))
    for grid in ((0, 8), (8, 0), (-2, 3)):
        with pytest.raises(ValueError):
            d.clahe(2.0, grid)


def test_uint8_chunk_of_more_than_2_31_voxels(torch):
    """64-bit indexing on both paths: the first and last sections, and the one that straddles byte 2^31."""
    from chunkflow_b200.chunk.device import DeviceChunk
    z, y, x = 2200, 1024, 1000
    assert z * y * x > 2 ** 31
    straddle = 2 ** 31 // (y * x)
    assert straddle * y * x < 2 ** 31 < (straddle + 1) * y * x
    a = lambda n, k: torch.arange(n, device="cuda", dtype=torch.int32).view(k)
    t = ((a(z, (z, 1, 1)) * 7 + a(y, (1, y, 1)) * 13 + a(x, (1, 1, x)) * 5 + a(y, (1, y, 1)) * a(x, (1, 1, x)) % 37) % 251).to(torch.uint8)
    d = DeviceChunk(t)
    for clip, grid in ((2.0, (8, 8)), (20.0, (512, 512))):
        out = d.clahe(clip, grid).tensor
        for k in (0, straddle, z - 1):
            np.testing.assert_array_equal(out[k].cpu().numpy(), CO.apply_section(t[k].cpu().numpy(), clip, grid), err_msg=f"{grid} {k}")
        del out
    del t, d
    torch.cuda.empty_cache()


def test_plugin_with_host_and_device_chunks(torch):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.plugins import clahe as plugin
    img = np.random.default_rng(9).integers(0, 256, (4, 120, 90), dtype=np.uint8)
    want = CO.clahe(img, plugin.clipLimit, plugin.tileGridSize)
    host = img.copy()
    view = host[2]
    c = Chunk(host, voxel_offset=(1, 2, 3), voxel_size=(40, 4, 4))
    assert plugin.execute(c) is c and c.array is host
    np.testing.assert_array_equal(host, want)
    np.testing.assert_array_equal(view, want[2])
    d = to_device(torch, img, voxel_offset=(5, 6, 7))
    tensor = d.tensor
    assert plugin.execute(d) is d and d.tensor is tensor
    assert isinstance(d, DeviceChunk) and tuple(d.voxel_offset) == (5, 6, 7)
    np.testing.assert_array_equal(d.tensor.cpu().numpy(), want)
    with pytest.raises(AssertionError):
        plugin.execute(to_device(torch, np.zeros((2, 3, 8, 8), np.float32)))


def test_cli_chains_on_host_and_device_chunks(torch):
    from click.testing import CliRunner
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.flow.cli import main, operator
    img = np.random.default_rng(5).integers(0, 256, (5, 70, 90), dtype=np.uint8)
    seen = {}

    @main.command("capture-clahe-test")
    @operator
    def capture(tasks):
        for task in tasks:
            seen.update(task)
            yield task
    try:
        @main.command("load-clahe-test")
        @operator
        def load(tasks):
            for task in tasks:
                task["img"] = Chunk(img.copy(), voxel_offset=(2, 4, 6), voxel_size=(40, 4, 4))
                yield task
        r = CliRunner().invoke(main, ["load-clahe-test", "clahe", "-i", "img", "-o", "eq",
                                      "clahe", "-i", "img", "-o", "eq8", "--clip-limit", "2", "--tile-grid-size", "8", "4",
                                      "to-device", "-i", "img", "-o", "dimg", "clahe", "-i", "dimg", "-o", "deq", "-c", "5", "-t", "18", "26",
                                      "to-host", "-i", "deq", "-o", "heq", "capture-clahe-test"], catch_exceptions=False)
        assert r.exit_code == 0, r.output
    finally:
        main.commands.pop("capture-clahe-test", None)
        main.commands.pop("load-clahe-test", None)
    assert isinstance(seen["eq"], Chunk) and tuple(seen["eq"].voxel_offset) == (2, 4, 6)
    assert tuple(seen["eq"].voxel_size) == (40, 4, 4)
    np.testing.assert_array_equal(seen["eq"].array, CO.clahe(img, 20.0, (512, 512)))
    np.testing.assert_array_equal(seen["eq8"].array, CO.clahe(img, 2.0, (8, 4)))
    np.testing.assert_array_equal(seen["img"].array, img)
    assert isinstance(seen["deq"], DeviceChunk) and tuple(seen["deq"].voxel_offset) == (2, 4, 6)
    np.testing.assert_array_equal(seen["heq"].array, CO.clahe(img, 5.0, (18, 26)))
