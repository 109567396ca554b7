"""`clahe` (DESIGN.md section 0, row f9) on the CPU: the numpy oracle (oracle/clahe_oracle.py) against live OpenCV and against
golden vectors of the reference's own plugin (tests/golden/clahe_reference.npz, made by tests/golden/make_golden_clahe.py);
the FMA negative control; csrc/clahe.cu, compiled for the host behind a one-lane CUDA shim (tests/host_emulation), against
the oracle on both paths; the refusals; the command's options."""
import ctypes as C
import os

import numpy as np
import pytest

import host_emulation
from oracle import clahe_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "clahe_reference.npz")
SMALL_TILE_MAX = 64   # kClaheSmallTileMax in csrc/clahe_kernels.cuh


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def golden_cases(gold):
    """(name, input, clip, (tiles_x, tiles_y), result)"""
    for key in sorted(k for k in gold if k.endswith("/in")):
        name = key[:-len("/in")]
        yield name, gold[key], float(gold[f"{name}/clip"]), tuple(int(v) for v in gold[f"{name}/grid"]), gold[f"{name}/out"]


def image(rng, shape, kind):
    if kind == "random":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "low":
        return rng.integers(60, 66, shape, dtype=np.uint8)
    z, y, x = shape
    yy, xx = np.mgrid[:y, :x]
    return np.broadcast_to(((np.sin(yy / 7.0) + np.cos(xx / 11.0)) * 60 + 128).astype(np.uint8), shape).copy()


# ------------------------------------------------------------------------------------------------------------
# the oracle against OpenCV and the reference
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1), (37, 129), (5, 700), (64, 64), (100, 90), (1, 50), (50, 1), (7, 3)])
def test_oracle_equals_live_cv2(shape):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(sum(shape))
    for grid in ((1, 1), (3, 5), (7, 3), (8, 8), (18, 26), (64, 2), (2, 64)):
        for clip in (0, 0.5, 1, 2, 3, 5, 20, 40, -1, 1e12):
            a = image(rng, (1,) + shape, ("random", "low", "smooth")[int(rng.integers(3))])[0]
            np.testing.assert_array_equal(CO.apply_section(a, clip, grid), cv2.createCLAHE(clip, grid).apply(a),
                                          err_msg=f"{shape} {grid} {clip}")


def test_oracle_equals_live_cv2_at_the_plugin_setting():
    cv2 = pytest.importorskip("cv2")
    a = np.random.default_rng(4).integers(0, 256, (300, 257), dtype=np.uint8)
    np.testing.assert_array_equal(CO.apply_section(a, 20.0, (512, 512)), cv2.createCLAHE(20.0, (512, 512)).apply(a))


def test_golden_covers_the_cases(gold):
    cases = {name: (a, clip, grid) for name, a, clip, grid, _ in golden_cases(gold)}
    assert str(gold["cv2_version"]).startswith("4.")
    assert cases["plugin_default"][1:] == (20.0, (512, 512))
    grids = {grid for _, clip, grid in cases.values()}
    assert {(8, 8), (18, 26), (512, 512)} <= grids
    clips = {clip for _, clip, _ in cases.values()}
    assert 0.0 in clips and min(clips) < 0 and max(clips) >= 1e12
    shapes = [a.shape for a, _, _ in cases.values()]
    assert all(len(s) == 3 and s[0] > 1 for s in shapes)
    assert any(s[1] == 1 for s in shapes) and any(s[2] == 1 for s in shapes)
    assert any(grid[0] > a.shape[2] and grid[1] > a.shape[1] for a, _, grid in cases.values())


def test_oracle_against_golden(gold):
    for name, a, clip, grid, want in golden_cases(gold):
        np.testing.assert_array_equal(CO.clahe(a, clip, grid), want, err_msg=name)


def test_fused_interpolation_differs_from_golden(gold):
    """Negative control: contracting the blend into FMAs changes pixels that the reference's output pins."""
    differing = 0
    for name, a, clip, grid, want in golden_cases(gold):
        if grid != (512, 512):
            differing += int((CO.clahe(a, clip, grid, fma=True) != want).sum())
    assert differing > 0


def test_oracle_against_the_live_reference():
    from oracle import clahe_harness as CH
    if not CH.available():
        pytest.skip("the reference tree or OpenCV is not available here (the golden vectors pin the oracle everywhere)")
    from chunkflow_b200.plugins import clahe as plugin
    assert CH.plugin_defaults() == (plugin.clipLimit, plugin.tileGridSize)
    a = image(np.random.default_rng(8), (2, 45, 77), "smooth")
    np.testing.assert_array_equal(CO.clahe(a, 2.0, (5, 3)), CH.clahe_plugin(a, 2.0, (5, 3)))


def test_oracle_refusals():
    with pytest.raises(TypeError):
        CO.clahe(np.zeros((2, 8, 8), np.uint16))
    with pytest.raises(ValueError):
        CO.clahe(np.zeros((3, 2, 8, 8), np.uint8))
    with pytest.raises(ValueError):
        CO.clahe(np.zeros((8, 8), np.uint8))
    for grid in ((0, 4), (4, 0), (-1, 1)):
        with pytest.raises(ValueError):
            CO.clahe(np.zeros((2, 8, 8), np.uint8), 2.0, grid)


# ------------------------------------------------------------------------------------------------------------
# the device code on the host (one-lane CUDA shim)
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("clahe", tmp_path_factory)
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    lib.cfb_clahe_workspace.argtypes = [i64, i64, i64, i32, i32, C.POINTER(i64)]
    lib.cfb_clahe_device.argtypes = [vp, vp, i64, i64, i64, C.c_double, i32, i32, vp, i64, vp]
    lib.emu_clahe_path.argtypes = [vp, vp, i64, i64, i64, C.c_double, i32, i32, C.c_int, i64]
    lib.emu_small_region.argtypes = [i64, i64, i64, i64, vp]
    return lib


def emu_clahe(lib, a, clip, grid, path=-1, batch=2, offset=0):
    """-> (result, path taken).  path -1: cfb_clahe_device with the workspace of cfb_clahe_workspace, which chooses the path
    and the batch (the small-tile path needs none); 0 / 1: the table path in batches of ``batch`` sections / the small-tile
    path.  ``offset`` bytes shift the input and (by 3) the output off 16-byte alignment."""
    src = np.zeros(a.size + 32, np.uint8)[offset:offset + a.size].reshape(a.shape)
    src[...] = a
    dst = np.zeros(a.size + 32, np.uint8)[3 if offset else 0:][:a.size].reshape(a.shape)
    p = lambda b: C.c_void_p(b.ctypes.data)
    if path < 0:
        need = C.c_int64()
        assert lib.cfb_clahe_workspace(*a.shape, grid[0], grid[1], C.byref(need)) == 0, lib.cfb_last_error()
        work = np.zeros(max(need.value, 1), np.uint8)
        rc = lib.cfb_clahe_device(p(src), p(dst), *a.shape, clip, grid[0], grid[1], p(work), need.value, None)
        path = int(need.value == 0)
    else:
        rc = lib.emu_clahe_path(p(src), p(dst), *a.shape, clip, grid[0], grid[1], path, batch)
    assert rc == 0, lib.cfb_last_error()
    return dst.copy(), path


def tile_pixels(y, x, grid):
    ph, pw, th, tw = CO.geometry(y, x, grid[0], grid[1])
    return th * tw


@pytest.mark.parametrize("shape", [(3, 37, 129), (2, 5, 70), (3, 1, 33), (3, 33, 1), (5, 64, 64), (2, 100, 90)])
@pytest.mark.parametrize("offset", [0, 5])
def test_emulated_paths_equal_the_oracle(emu, shape, offset):
    """Both paths on the same inputs, table batches of 2 sections (that do not divide z), aligned and unaligned buffers."""
    rng = np.random.default_rng(sum(shape) + offset)
    for grid in ((1, 1), (3, 5), (8, 8), (18, 26), (64, 2), (7, 3), (40, 40)):
        for clip in (0, 2, 20, -1, 1e12):
            a = image(rng, shape, ("random", "low", "smooth")[int(rng.integers(3))])
            want = CO.clahe(a, clip, grid)
            for path in (0, 1):
                got, taken = emu_clahe(emu, a, clip, grid, path, batch=2, offset=offset)
                assert taken == path
                np.testing.assert_array_equal(got, want, err_msg=f"{shape} {grid} {clip} path {path}")


def test_emulated_path_selection_at_the_threshold(emu):
    """The library's choice: tiles of at most SMALL_TILE_MAX pixels take the small-tile path, larger ones the table."""
    rng = np.random.default_rng(5)
    seen = set()
    for y, x, grid in ((64, 64, (8, 8)), (64, 64, (8, 4)), (64, 64, (4, 8)), (64, 64, (16, 8)), (64, 64, (32, 32)),
                       (66, 64, (2, 32)), (64, 33, (1, 2)), (130, 64, (2, 64))):
        a = image(rng, (3, y, x), "random")
        t = tile_pixels(y, x, grid)
        got, taken = emu_clahe(emu, a, 3.0, grid, batch=1)
        assert taken == (1 if t <= SMALL_TILE_MAX else 0), (y, x, grid, t)
        seen.add((t, taken))
        np.testing.assert_array_equal(got, CO.clahe(a, 3.0, grid), err_msg=f"{grid}")
    assert (SMALL_TILE_MAX, 1) in seen and any(t > SMALL_TILE_MAX and p == 0 for t, p in seen)


def test_emulated_against_golden(emu, gold):
    for name, a, clip, grid, want in golden_cases(gold):
        got, _ = emu_clahe(emu, a, clip, grid, batch=1)
        np.testing.assert_array_equal(got, want, err_msg=name)


def test_small_tile_regions_fit_shared_memory(emu):
    """Regions shrink until the staged tiles fit 48 KiB, down to one tile."""
    out = (C.c_int64 * 4)()
    for y, x, grid in ((1024, 1024, (512, 512)), (64, 1024, (1024, 2)), (1024, 64, (2, 1024)), (1024, 1024, (256, 128)),
                       (1024, 1024, (32, 1024))):
        emu.emu_small_region(y, x, grid[0], grid[1], out)
        ry, rx, th, tw = list(out)
        slots = (ry + 2) * (rx + 2)
        assert ry >= 1 and rx >= 1 and slots * th * tw * 3 + slots * 24 <= 48 << 10, (grid, ry, rx)


# ------------------------------------------------------------------------------------------------------------
# the bindings and the command
# ------------------------------------------------------------------------------------------------------------
def test_wrappers_validate_before_the_library_is_touched(monkeypatch):
    from chunkflow_b200 import _native
    monkeypatch.setattr(_native, "load", lambda: pytest.fail("the native library must not be reached"))
    with pytest.raises(ValueError):
        _native.clahe_workspace((3, 4, 8, 8), (8, 8))
    with pytest.raises(ValueError):
        _native.clahe_workspace((4, 8), (8, 8))
    for grid in ((0, 8), (8, 0), (8,)):
        with pytest.raises(ValueError):
            _native.clahe_device(16, 1 << 40, (4, 8, 8), 2.0, grid, 0, 0)


def test_native_refusals_need_no_device():
    """Tile grids, sizes, overlaps and workspaces are refused by the library before any CUDA call (fake device addresses)."""
    from chunkflow_b200 import _native
    if not os.path.exists(os.path.join(ROOT, "chunkflow_b200", "_native", "libchunkflow_b200.so")):
        pytest.skip("the native library is not built")
    assert _native.clahe_workspace((10, 1024, 1024), (8, 8)) == 10 * 64 * 256          # 64 LUTs of 256 bytes per section
    assert _native.clahe_workspace((3000, 1024, 1024), (8, 8)) == 2048 * 64 * 256      # batches of 2048 sections: 32 MiB
    assert _native.clahe_workspace((10, 1024, 1024), (512, 512)) == 0                  # 4-pixel tiles: no table
    lib = _native.load()
    out = C.c_int64()
    assert lib.cfb_clahe_workspace(4, 8, 8, 0, 8, C.byref(out)) == _native.ERR_INVALID_ARGUMENT
    assert b"tile" in lib.cfb_last_error()
    assert lib.cfb_clahe_workspace(1, 8, (1 << 24) + 1, 8, 8, C.byref(out)) == _native.ERR_INVALID_ARGUMENT
    assert lib.cfb_clahe_workspace(1, 50000, 50000, 8, 8, C.byref(out)) == _native.ERR_INVALID_ARGUMENT
    assert b"2^31 - 1" in lib.cfb_last_error()
    dev = lambda a: C.c_void_p(a)
    assert lib.cfb_clahe_device(dev(1 << 40), dev((1 << 40) + 100), 2, 16, 16, 2.0, 8, 8, None, 0, None) == _native.ERR_INVALID_ARGUMENT
    assert b"overlap" in lib.cfb_last_error()
    assert lib.cfb_clahe_device(dev(1 << 40), dev(1 << 41), 2, 1024, 1024, 2.0, 8, 8, None, 0, None) == _native.ERR_INVALID_ARGUMENT
    assert b"workspace" in lib.cfb_last_error()
    assert lib.cfb_clahe_device(dev(1 << 40), dev(1 << 41), 2, 1024, 1024, 2.0, 8, 8, dev(1 << 42), 100, None) == _native.ERR_INVALID_ARGUMENT
    assert b"smaller" in lib.cfb_last_error()
    assert lib.cfb_clahe_device(dev(1 << 40), dev(1 << 41), 2, 1024, 1024, 2.0, 8, 8, dev((1 << 41) + 4096), 1 << 20,
                                None) == _native.ERR_INVALID_ARGUMENT
    assert b"overlaps" in lib.cfb_last_error()


def test_plugin_module_matches_the_reference_constants():
    from chunkflow_b200.plugins import clahe as plugin
    assert plugin.clipLimit == 20.0 and tuple(plugin.tileGridSize) == (512, 512)
    with pytest.raises(AssertionError):
        from chunkflow_b200.chunk import Chunk
        plugin.execute(Chunk(np.zeros((3, 4, 8, 8), np.uint8)))


def test_command_options():
    from chunkflow_b200.flow.cli import main
    p = {q.name: q for q in main.commands["clahe"].params}
    assert set(p) == {"input_chunk_name", "output_chunk_name", "clip_limit", "tile_grid_size"}
    assert p["input_chunk_name"].opts == ["--input-chunk-name", "-i"] and p["output_chunk_name"].opts == ["--output-chunk-name", "-o"]
    assert p["clip_limit"].opts == ["--clip-limit", "-c"] and p["clip_limit"].default == 20.0
    assert p["tile_grid_size"].opts == ["--tile-grid-size", "-t"] and p["tile_grid_size"].nargs == 2
    assert tuple(p["tile_grid_size"].default) == (512, 512)
