"""`gaussian-filter` and the median filter (DESIGN.md section 0, row f8) on the CPU: the numpy oracle (oracle/filters_oracle.py)
against live scipy.ndimage and against golden vectors of the reference's own three callers (tests/golden/filters_reference.npz,
made by tests/golden/make_golden_filters.py); csrc/filters.cu, compiled for the host behind a one-lane CUDA shim
(tests/host_emulation), against the oracle; the refusals; the command's options."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy import ndimage as ndi

import host_emulation
from oracle import filters_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "filters_reference.npz")
MODES = tuple(FO.MODES)
SIGMAS = (0, 0.1, 0.5, 1, 2, 3.7, (0, 1), (1, 2))
MEDIAN_SIZES = ((3, 1, 1), (1, 3, 3), (3, 3, 3), (2, 2, 2), (5, 5, 5), (4, 1, 2), (1, 5, 1), (1, 2, 3), 1, 3)


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def golden_cases(gold):
    """(name, caller, input, keyword arguments, result)"""
    for key in sorted(k for k in gold if k.endswith("/caller")):
        name = key[:-len("/caller")]
        caller = str(gold[key])
        if caller == "median_plugin":
            size = gold[f"{name}/size"]
            kw = {"size": int(size) if size.ndim == 0 else tuple(int(v) for v in size), "mode": str(gold[f"{name}/mode"])}
        else:
            sigma = gold[f"{name}/sigma"]
            kw = {"sigma": float(sigma) if sigma.ndim == 0 else tuple(float(v) for v in sigma)}
        yield name, caller, gold[f"{name}/in"], kw, gold[f"{name}/out"]


def oracle_call(caller, arr, kw):
    if caller == "method":
        return FO.gaussian_filter_2d(arr, kw["sigma"])
    if caller == "gaussian_plugin":
        return FO.gaussian_plugin(arr, kw["sigma"])
    return FO.median_filter(arr, kw["size"], kw["mode"])


def image(rng, shape, dtype):
    if np.dtype(dtype) == np.uint8:
        return rng.integers(0, 256, shape, dtype=np.uint8)
    return (rng.random(shape) * 100).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------
# the oracle against scipy and the reference
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("shape", [(1, 7), (2, 5), (3, 9), (9, 1), (9, 2), (8, 40), (13, 17), (3, 6, 7)])
def test_gaussian_oracle_equals_scipy(dtype, shape):
    """Lines shorter than the radius included (sigma 3.7: radius 15)."""
    a = image(np.random.default_rng(sum(shape)), shape, dtype)
    for s in SIGMAS + (0.5 * np.arange(1, len(shape) + 1),):
        if np.ndim(s) and len(s) != len(shape):
            continue
        np.testing.assert_array_equal(FO.gaussian_filter(a, s), ndi.gaussian_filter(a, s), err_msg=str(s))


@pytest.mark.parametrize("value", [0, 128, 255])
def test_gaussian_oracle_on_constant_images(value):
    """Weights that sum to just below 1 and truncation: a constant 128 comes back as 127 from scipy, and from the oracle."""
    a = np.full((20, 30), value, np.uint8)
    for s in (0.5, 1, 2, 3.7):
        np.testing.assert_array_equal(FO.gaussian_filter(a, s), ndi.gaussian_filter(a, s))


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 2, 3), (2, 2, 2), (3, 1, 2), (5, 4, 6), (2, 7, 3)])
def test_median_oracle_equals_scipy_in_every_mode(dtype, shape):
    """Length-1 and length-2 axes in every mode (mirror on length 1 is a special case in scipy)."""
    a = np.random.default_rng(sum(shape)).integers(0, 5, shape).astype(dtype)
    for mode in MODES:
        for size in MEDIAN_SIZES:
            np.testing.assert_array_equal(FO.median_filter(a, size, mode), ndi.median_filter(a, size=size, mode=mode),
                                          err_msg=f"{mode} {size}")


def test_golden_covers_the_three_callers(gold):
    cases = list(golden_cases(gold))
    assert {c for _, c, *_ in cases} == {"method", "gaussian_plugin", "median_plugin"}
    assert {a.shape[0] for _, c, a, *_ in cases if c == "method" and a.ndim == 4} == {3, 4}
    assert {kw["mode"] for _, c, _, kw, _ in cases if c == "median_plugin"} == set(MODES)


def test_oracle_against_golden(gold):
    for name, caller, arr, kw, want in golden_cases(gold):
        out = oracle_call(caller, arr, kw)
        assert out.dtype == want.dtype, name
        np.testing.assert_array_equal(out, want, err_msg=name)


def test_command_on_4d_chunks_filters_across_channels(gold):
    """The reference's quirk, kept: on (c,z,y,x) its result is the 3-D (c,y,x) filter of every z, not the per-channel one."""
    for name, caller, arr, kw, want in golden_cases(gold):
        if caller == "method" and arr.ndim == 4 and np.ndim(kw["sigma"]) == 0:
            assert not np.array_equal(want, FO.gaussian_plugin(arr, kw["sigma"])), name
            want3 = np.stack([ndi.gaussian_filter(arr[:, z], kw["sigma"]) for z in range(arr.shape[1])], axis=1)
            np.testing.assert_array_equal(want, want3, err_msg=name)


def test_oracle_against_the_live_reference():
    from oracle import filters_harness as FH
    if not FH.available():
        pytest.skip("the reference tree is not available here (the golden vectors pin the oracle everywhere)")
    rng = np.random.default_rng(11)
    aff = rng.random((3, 2, 15, 18), dtype=np.float32)
    np.testing.assert_array_equal(FO.gaussian_filter_2d(aff, 2), FH.gaussian_filter_2d(aff, 2))
    np.testing.assert_array_equal(FO.gaussian_plugin(aff, 2), FH.gaussian_plugin(aff, 2))
    img = rng.integers(0, 256, (4, 15, 18), dtype=np.uint8)
    np.testing.assert_array_equal(FO.gaussian_filter_2d(img, 1), FH.gaussian_filter_2d(img, 1))
    np.testing.assert_array_equal(FO.median_filter(img, (3, 1, 1)), FH.median_plugin(img, (3, 1, 1)))


def test_oracle_refusals():
    with pytest.raises(TypeError):
        FO.gaussian_filter(np.zeros((4, 4), np.uint16), 1)
    with pytest.raises(TypeError):
        FO.median_filter(np.zeros((4, 4, 4), np.float64))
    with pytest.raises(ValueError, match="64"):
        FO.gaussian_filter(np.zeros((4, 4), np.uint8), 16.2)    # radius int(65.3) = 65
    FO.gaussian_filter(np.zeros((4, 4), np.uint8), 16)          # radius int(64.5) = 64, the largest
    with pytest.raises(ValueError, match="125"):
        FO.median_filter(np.zeros((4, 4, 4), np.uint8), (6, 5, 5))
    with pytest.raises(RuntimeError, match="sequence argument"):
        FO.median_filter(np.zeros((4, 4, 4), np.uint8), (3, 1))
    with pytest.raises(RuntimeError, match="sequence argument"):
        ndi.median_filter(np.zeros((4, 4, 4), np.uint8), (3, 1))


# ------------------------------------------------------------------------------------------------------------
# the device code on the host (one-lane CUDA shim)
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("filters", tmp_path_factory)
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    lib.emu_gaussian.argtypes = [i32, vp, i64, i64, i64, i64, vp, i32, vp, i32, vp, i32, i64]
    lib.cfb_median_filter_device.argtypes = [vp, i32, i64, i64, i64, i64, vp, i32, vp, vp]
    lib.emu_median_path.argtypes = [vp]
    return lib


def emu_gaussian(lib, arr, weights, batch):
    """weights: (c, y, x), each an array or None."""
    a = np.ascontiguousarray(arr).copy()
    czyx = (1,) + a.shape if a.ndim == 3 else a.shape
    keep = [None if w is None else np.ascontiguousarray(w, np.float64) for w in weights]
    args = []
    for w in keep:
        args += [None, 0] if w is None else [C.c_void_p(w.ctypes.data), len(w) - 1]
    rc = lib.emu_gaussian(0 if a.dtype == np.uint8 else 1, C.c_void_p(a.ctypes.data), *czyx, *args, batch)
    assert rc == 0, lib.cfb_last_error()
    return a


def weights_of(sigma, n):
    return [None if w is None else w for w in FO.axis_weights(sigma, n)]


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("shape", [(3, 37, 70), (2, 1, 9), (2, 2, 9), (2, 3, 9), (2, 9, 1), (2, 9, 2), (5, 33, 65), (1, 64, 128)])
@pytest.mark.parametrize("batch", [1, 2, 64])
def test_emulated_gaussian_equals_the_oracle(emu, dtype, shape, batch):
    """Shapes that are no multiple of the 32 x 64 tile, lines shorter than the radius, batches that do not divide z."""
    a = image(np.random.default_rng(shape[1] * shape[2]), shape, dtype)
    for s in SIGMAS:
        got = emu_gaussian(emu, a, [None] + weights_of(s, 2), batch)
        np.testing.assert_array_equal(got, FO.gaussian_filter_2d(a, s), err_msg=str(s))


@pytest.mark.parametrize("channels", [1, 3, 4])
@pytest.mark.parametrize("batch", [1, 3])
def test_emulated_gaussian_on_4d_chunks(emu, channels, batch):
    """The command (channel pass first) and the plugin (every (y,x) plane on its own)."""
    a = np.random.default_rng(channels).random((channels, 4, 21, 70), dtype=np.float32)
    for s in (1, (1, 0.5, 2), (0, 1, 1), 3.7):
        got = emu_gaussian(emu, a, weights_of(s, 3), batch)
        np.testing.assert_array_equal(got, FO.gaussian_filter_2d(a, s), err_msg=str(s))
    got = emu_gaussian(emu, a, [None] + weights_of(1.5, 2), batch)
    np.testing.assert_array_equal(got, FO.gaussian_plugin(a, 1.5))


def test_emulated_gaussian_at_the_largest_radius(emu):
    a = image(np.random.default_rng(3), (2, 40, 150), np.uint8)
    got = emu_gaussian(emu, a, [None] + weights_of(15.9, 2), 1)
    np.testing.assert_array_equal(got, FO.gaussian_filter_2d(a, 15.9))


def emu_median(lib, arr, size, mode):
    a = np.ascontiguousarray(arr)
    czyx = (1,) + a.shape if a.ndim == 3 else a.shape
    ext = FO.per_axis(size, a.ndim, "size")
    s = np.array(([1] + ext) if a.ndim == 3 else ext, np.int64)
    out = np.zeros_like(a)
    rc = lib.cfb_median_filter_device(C.c_void_p(a.ctypes.data), 0 if a.dtype == np.uint8 else 1, *czyx, C.c_void_p(s.ctypes.data),
                                      FO.MODES[mode], C.c_void_p(out.ctypes.data), None)
    assert rc == 0, lib.cfb_last_error()
    return out, lib.emu_median_path(C.c_void_p(s.ctypes.data))


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 1, 2), (1, 2, 5), (4, 2, 1), (7, 11, 13), (2, 3, 5, 6)])
def test_emulated_median_equals_the_oracle(emu, dtype, shape):
    a = np.random.default_rng(sum(shape)).integers(0, 6, shape).astype(dtype)
    if dtype == np.float32:
        a[a == 5] = np.inf
    paths = set()
    for mode in MODES:
        for size in MEDIAN_SIZES if len(shape) == 3 else ((1, 3, 1, 1), (2, 2, 2, 2), 2, (1, 1, 5, 5)):
            got, path = emu_median(emu, a, size, mode)
            paths.add(path)
            np.testing.assert_array_equal(got, FO.median_filter(a, size, mode), err_msg=f"{mode} {size}")
    assert paths == ({-1, 4, 16, 32, 0} if len(shape) == 3 else {-1, 16, 32})


# ------------------------------------------------------------------------------------------------------------
# the bindings and the command
# ------------------------------------------------------------------------------------------------------------
def test_wrappers_validate_before_the_library_is_touched(monkeypatch):
    from chunkflow_b200 import _native
    monkeypatch.setattr(_native, "load", lambda: pytest.fail("the native library must not be reached"))
    with pytest.raises(TypeError):
        _native.gaussian_filter_workspace(_native.DTYPE_U32, (4, 4, 4))
    with pytest.raises(ValueError):
        _native.gaussian_filter_workspace(_native.DTYPE_U8, (4, 4))
    with pytest.raises(ValueError, match="64"):
        _native.gaussian_filter_device(16, _native.DTYPE_U8, (4, 4, 4), [np.ones(66), None], 32, 64)
    with pytest.raises(ValueError):
        _native.gaussian_filter_device(16, _native.DTYPE_U8, (4, 4, 4), [None, None, None], 32, 64)
    with pytest.raises(TypeError):
        _native.median_filter_device(16, _native.DTYPE_U64, (4, 4, 4), (3, 1, 1), "reflect", 32)
    with pytest.raises(ValueError):
        _native.median_filter_device(16, _native.DTYPE_U8, (4, 4, 4), (3, 1), "reflect", 32)
    with pytest.raises(ValueError):
        _native.median_filter_device(16, _native.DTYPE_U8, (4, 4, 4), (3, 1, 1), "edge", 32)


def test_native_refusals_need_no_device():
    """Radius, window and dtype are refused by the library before any CUDA call (fake device addresses)."""
    from chunkflow_b200 import _native
    if not os.path.exists(os.path.join(ROOT, "chunkflow_b200", "_native", "libchunkflow_b200.so")):
        pytest.skip("the native library is not built")
    n = _native.gaussian_filter_workspace(_native.DTYPE_F32, (3, 100, 64, 64))
    assert n == 3 * 64 * 64 * 4 * 100            # 100 sections of 48 KiB fit the 32 MiB target
    assert _native.gaussian_filter_workspace(_native.DTYPE_F32, (3, 8, 2048, 2048)) == 3 * 2048 * 2048 * 4   # one section
    lib = _native.load()
    w = (C.c_double * 66)(*([1.0] * 66))
    assert lib.cfb_gaussian_filter_device(C.c_void_p(16), _native.DTYPE_U8, 1, 4, 4, 4, None, 0, w, 65, None, 0,
                                          C.c_void_p(1 << 40), 1 << 20, None) == _native.ERR_INVALID_ARGUMENT
    assert b"radius" in lib.cfb_last_error()
    size = (C.c_int64 * 4)(1, 6, 5, 5)
    assert lib.cfb_median_filter_device(C.c_void_p(16), _native.DTYPE_U8, 1, 8, 8, 8, C.byref(size), 0, C.c_void_p(1 << 40),
                                        None) == _native.ERR_INVALID_ARGUMENT
    assert b"125" in lib.cfb_last_error()
    size = (C.c_int64 * 4)(1, 3, 1, 1)
    assert lib.cfb_median_filter_device(C.c_void_p(16), _native.DTYPE_U32, 1, 8, 8, 8, C.byref(size), 0, C.c_void_p(1 << 40),
                                        None) == _native.ERR_INVALID_ARGUMENT


def test_gaussian_weights_are_the_oracles():
    from chunkflow_b200.chunk.device import gaussian_weights
    for s in (0.1, 0.5, 1, 2, 3.7, 15.9):
        np.testing.assert_array_equal(gaussian_weights(s), FO.gaussian_weights(s))


def test_command_options_are_spelled_like_the_reference():
    from chunkflow_b200.flow.cli import main
    g = {p.name: p for p in main.commands["gaussian-filter"].params}
    assert set(g) == {"name", "input_chunk_name", "sigma"}
    assert g["sigma"].opts == ["--sigma", "-s"] and g["sigma"].default == 1 and g["input_chunk_name"].opts == ["--input-chunk-name", "-i"]
    m = {p.name: p for p in main.commands["median-filter"].params}
    assert set(m) == {"input_chunk_name", "output_chunk_name", "size", "mode"}
    assert tuple(m["size"].default) == (3, 1, 1) and m["mode"].default == "reflect"
