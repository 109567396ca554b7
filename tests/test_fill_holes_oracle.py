"""`fill-segmentation-holes` on the CPU: the oracle's binary rule against live scipy.ndimage.binary_fill_holes, the oracle's
own properties (idempotence, keep-enclosed changes only zeros, nothing enclosed after remove-enclosed, nested enclosers), and
csrc/fill_holes.cu, compiled for the host behind the one-lane CUDA shim (tests/host_emulation), against the oracle for every
mode and dtype."""
import numpy as np
import pytest
from scipy import ndimage

import host_emulation
from chunkflow_b200 import _native as N
from oracle import fill_holes_oracle as F


def ball(shape, centre, radius):
    z, y, x = np.indices(shape)
    return (z - centre[0]) ** 2 + (y - centre[1]) ** 2 + (x - centre[2]) ** 2 <= radius ** 2


def shells(shape=(21, 22, 23)):
    """A ball in a gap in a shell in a gap in a shell, all around one centre: ids 7 (ball), 5 (inner shell), 3 (outer)."""
    c = tuple((s - 1) / 2 for s in shape)
    seg = np.zeros(shape, np.uint32)
    seg[ball(shape, c, 9.5) & ~ball(shape, c, 8)] = 3
    seg[ball(shape, c, 6.5) & ~ball(shape, c, 5)] = 5
    seg[ball(shape, c, 3)] = 7
    seg[ball(shape, c, 1)] = 0                     # a bubble inside the ball
    return seg


def hollow_boxes(shape, seed, n=6):
    """Boxes with carved cavities, some of them cut by a chunk face, some holding a smaller object."""
    rng = np.random.default_rng(seed)
    seg = np.zeros(shape, np.uint32)
    for k in range(1, n + 1):
        lo = rng.integers(-2, np.array(shape) - 4)
        hi = lo + rng.integers(5, 10, 3)
        lo, hi = np.maximum(lo, 0), np.minimum(hi, shape)
        box = tuple(slice(a, b) for a, b in zip(lo, hi))
        seg[box] = 11 * k
        inner = tuple(slice(a + 1, b - 1) for a, b in zip(lo, hi))
        seg[inner] = 0
        if rng.random() < 0.5:
            mid = tuple(slice((a + b) // 2, (a + b) // 2 + 1) for a, b in zip(lo, hi))
            seg[mid] = 11 * k + 3
    return seg


def diagonal_walls(shape=(11, 12, 13)):
    """A diamond shell |dz| + |dy| + |dx| == 4 of id 1, whose voxels touch only along edges and corners: it blocks a 6-connected
    flood of the background (a face step changes the sum by one), so binary mode fills it, but each of its voxels is an object
    of its own and encloses nothing.  Next to it, a staircase wall of id 2 across the whole chunk."""
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, np.uint32)
    seg[np.abs(z - 5) + np.abs(y - 5) + np.abs(x - 5) == 4] = 1
    seg[y - x == 6] = 2
    return seg


def salt_and_pepper(shape, seed, k=3):
    return np.random.default_rng(seed).integers(0, k, shape).astype(np.uint32)


VOLUMES = {
    "shells": shells(),
    "hollow_boxes": hollow_boxes((18, 20, 22), 1),
    "hollow_boxes_2": hollow_boxes((16, 17, 19), 2, 9),
    "diagonal_walls": diagonal_walls(),
    "salt_and_pepper": salt_and_pepper((12, 13, 14), 3),
    "sparse_noise": (np.random.default_rng(4).random((10, 12, 14)) < 0.6).astype(np.uint32) * 9,
    "all_zero": np.zeros((5, 6, 7), np.uint32),
    "single_id": np.full((5, 6, 7), 42, np.uint32),
    "one_slice": shells((1, 22, 23)),
    "one_row": salt_and_pepper((1, 1, 40), 5, 2),
    "one_column": shells((21, 1, 23)),
}


def test_binary_is_live_scipy():
    for seed in range(8):
        rng = np.random.default_rng(seed)
        arr = (rng.random((14, 15, 16)) < 0.45 + 0.05 * seed).astype(np.uint8) * rng.integers(1, 9)
        out, n = F.fill(arr, "binary")
        want = ndimage.binary_fill_holes(arr != 0)
        assert out.dtype == arr.dtype and np.array_equal(out, want.astype(np.uint8)) and n == int((want & (arr == 0)).sum())


def test_float32_zero_signs_and_nan():
    arr = np.zeros((5, 5, 5), np.float32)
    arr[1:4, 1:4, 1:4] = np.nan
    arr[2, 2, 2] = -0.0
    out, n = F.fill(arr, "binary")
    assert n == 1 and out.dtype == np.float32
    assert out[2, 2, 2] == 1 and out[0, 0, 0] == 0 and out[1, 1, 1] == 1 and set(np.unique(out)) == {0, 1}


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_oracle_properties(name):
    seg = VOLUMES[name]
    for mode in F.MODES:
        once, _ = F.fill(seg, mode)
        twice, n2 = F.fill(once, mode)
        assert np.array_equal(once, twice), mode
        if mode == "binary":
            assert n2 == 0
    keep, _ = F.fill(seg, "keep-enclosed")
    assert np.array_equal(keep[seg != 0], seg[seg != 0])
    removed, _ = F.fill(seg, "remove-enclosed")
    assert all(not e.any() for _, _, e in F.objects(removed))


def test_diagonal_walls_block_the_background_but_enclose_nothing():
    seg = diagonal_walls()
    assert F.fill(seg, "binary")[1] == 1 + 6 + 18 + 38   # the voxels with |dz| + |dy| + |dx| <= 3
    for mode in F.MODES[1:]:
        assert F.fill(seg, mode)[1] == 0


def test_shells_nest_and_each_mode_fills_its_own_way():
    seg = shells()
    c = tuple(s // 2 for s in seg.shape)
    assert [v for v, _ in F.enclosers(seg, c)] == [7, 5, 3]             # the bubble: inside the ball, the inner and outer shells
    gap = (c[0], c[1], c[2] + 4)                                          # between the ball and the inner shell
    assert seg[gap] == 0 and [v for v, _ in F.enclosers(seg, gap)] == [5, 3]
    keep, _ = F.fill(seg, "keep-enclosed")
    assert keep[c] == 7 and keep[gap] == 5 and keep[c[0], c[1], c[2] + 7] == 3
    removed, _ = F.fill(seg, "remove-enclosed")
    assert removed[c] == 3 and removed[gap] == 3 and set(np.unique(removed)) == {0, 3}


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_enclosers_are_nested(name):
    seg = VOLUMES[name]
    objs = F.objects(seg)
    for i, (_, si, ei) in enumerate(objs):
        for _, sj, ej in objs[i + 1:]:
            both = ei & ej
            if both.any():   # the smaller filled mask lies inside the larger one
                small, large = (ei, ej) if si < sj else (ej, ei)
                assert si != sj and not (small & ~large).any()


# ---- the host emulation of csrc/fill_holes.cu against the oracle ----
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("fill_holes", tmp_path_factory)
    N.bind_fill_holes(lib)
    return lib


def code_of(arr):
    return {1: N.DTYPE_U8, 8: N.DTYPE_U64}.get(arr.itemsize, N.DTYPE_F32 if arr.dtype == np.float32 else N.DTYPE_U32)


def emu_fill(lib, arr, mode, slots=1 << 6, stats=None):
    """DeviceChunk.fill_holes's sequence on host buffers: components, then (per object) the graph, grown while the table is too
    full, and the enclosure, then the apply pass."""
    arr = np.ascontiguousarray(arr)
    code = code_of(arr)
    work = np.zeros(N.fill_holes_workspace(arr.shape, lib=lib), np.uint8)
    comps = N.fill_holes_components_device(arr.ctypes.data, code, arr.shape, mode, work.ctypes.data, lib=lib)
    if stats is not None:
        stats.update(components=comps, retries=0)
    if mode != "binary":
        while True:
            table = np.zeros(N.fill_holes_table_workspace(slots, lib=lib), np.uint8)
            try:
                edges = N.fill_holes_graph_device(work.ctypes.data, arr.shape, table.ctypes.data, slots, lib=lib)
                break
            except N.NativeError as err:
                assert err.code == N.ERR_CAPACITY and "pair table" in str(err)
                slots <<= 2
                if stats is not None:
                    stats["retries"] += 1
        if stats is not None:
            stats["edges"] = edges
        N.fill_holes_enclose(work.ctypes.data, arr.shape, table.ctypes.data, slots, edges, lib=lib)
    out = np.empty_like(arr)
    n = N.fill_holes_apply_device(arr.ctypes.data, code, arr.shape, work.ctypes.data, out.ctypes.data, lib=lib)
    return out, n


def as_dtype(seg, dtype):
    """``seg`` in ``dtype``; ids of the 64-bit types moved beyond 2^32, int64 ones made negative."""
    if dtype in (np.uint64, np.int64):
        ids = seg.astype(np.uint64)
        ids[ids != 0] += np.uint64(2 ** 32 + 5)
        return ids.view(np.int64) * -1 if dtype == np.int64 else ids
    if dtype == np.int32:
        return seg.astype(np.int64).astype(np.int32) * -1
    return seg.astype(dtype)


@pytest.mark.parametrize("mode", F.MODES)
@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_emulation_equals_the_oracle(emu, name, mode):
    dtypes = F.BINARY_DTYPES if mode == "binary" else F.OBJECT_DTYPES
    for dtype in dtypes:
        seg = VOLUMES[name]
        arr = (seg != 0) if dtype is np.bool_ else (seg % 251).astype(np.float32) if dtype is np.float32 else as_dtype(seg, dtype)
        want, n = F.fill(arr, mode)
        got, m = emu_fill(emu, arr, mode)
        assert got.dtype == arr.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)) and m == n, (dtype, m, n)


def test_emulation_float_signs_and_nan(emu):
    arr = np.zeros((6, 7, 8), np.float32)
    arr[1:5, 1:6, 1:7] = np.nan
    arr[2:4, 2:5, 2:6] = -0.0
    arr[3, 3, 3] = 0.5
    want, n = F.fill(arr, "binary")
    got, m = emu_fill(emu, arr, "binary")
    assert np.array_equal(got, want) and m == n == 2 * 3 * 4 - 1 and np.array_equal(ndimage.binary_fill_holes(arr != 0), got == 1)


def test_emulation_retries_a_full_table(emu):
    seg = salt_and_pepper((10, 11, 12), 6, 4)
    st = {}
    got, m = emu_fill(emu, seg, "remove-enclosed", slots=2, stats=st)
    want, n = F.fill(seg, "remove-enclosed")
    assert st["retries"] >= 3 and st["edges"] > 100 and np.array_equal(got, want) and m == n


def test_emulation_refuses_bad_arguments(emu):
    arr = shells()
    work = np.zeros(N.fill_holes_workspace(arr.shape, lib=emu), np.uint8)
    for code, mode in ((N.DTYPE_U8, "keep-enclosed"), (N.DTYPE_F32, "remove-enclosed"), (N.DTYPE_BOOL, "binary")):
        with pytest.raises(N.NativeError, match="fill holes: .*take"):
            N.fill_holes_components_device(arr.ctypes.data, code, arr.shape, mode, work.ctypes.data, lib=emu)
    with pytest.raises(ValueError, match="mode"):
        N.fill_holes_components_device(arr.ctypes.data, N.DTYPE_U32, arr.shape, "holes", work.ctypes.data, lib=emu)
    with pytest.raises(N.NativeError, match="2\\^32 voxels"):
        N.fill_holes_workspace((1 << 11, 1 << 11, 1 << 10), lib=emu)
    with pytest.raises(N.NativeError, match="power of two"):
        N.fill_holes_table_workspace(1 << 31, lib=emu)
    N.fill_holes_components_device(arr.ctypes.data, N.DTYPE_U32, arr.shape, "binary", work.ctypes.data, lib=emu)
    table = np.zeros(N.fill_holes_table_workspace(64, lib=emu), np.uint8)
    with pytest.raises(N.NativeError, match="binary mode needs no"):
        N.fill_holes_graph_device(work.ctypes.data, arr.shape, table.ctypes.data, 64, lib=emu)
    N.fill_holes_components_device(arr.ctypes.data, N.DTYPE_U32, arr.shape, "keep-enclosed", work.ctypes.data, lib=emu)
    out = np.empty_like(arr)
    with pytest.raises(N.NativeError, match="after cfb_fill_holes_enclose"):
        N.fill_holes_apply_device(arr.ctypes.data, N.DTYPE_U32, arr.shape, work.ctypes.data, out.ctypes.data, lib=emu)


def test_oracle_refuses_other_dtypes_and_modes():
    with pytest.raises(TypeError, match="keep-enclosed mode takes"):
        F.fill(np.zeros((2, 2, 2), np.uint8), "keep-enclosed")
    with pytest.raises(TypeError, match="binary mode takes"):
        F.fill(np.zeros((2, 2, 2), np.float64), "binary")
    with pytest.raises(ValueError):
        F.fill(np.zeros((2, 2, 2), np.uint32), "fill")
