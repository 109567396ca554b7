"""`downsample` (DESIGN.md section 0, row f7; reference flow/flow.py:1545-1573, lib/igneous/downsample.py) on the CPU: the numpy
oracle (oracle/downsample_oracle.py) against golden vectors of the REAL vendored downsampler
(tests/golden/downsample_reference.npz, made by tests/golden/make_golden_downsample.py) and, where the reference tree exists,
against the live module; csrc/downsample.cu, compiled for the host behind a one-lane CUDA shim (tests/host_emulation),
against the oracle; the command's option names; the wrappers' argument checks."""
import ctypes as C
import itertools
import os
import re

import numpy as np
import pytest

import host_emulation
from conftest import has_gpu
from oracle import downsample_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "downsample_reference.npz")
KINDS = {np.dtype(bool): 0, np.dtype(np.uint32): 1, np.dtype(np.uint64): 2, np.dtype(np.int64): 2}


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def golden_cases(gold):
    """(name, kind, input, factor, raises, raises with factor // 2, result or None)"""
    for key in sorted(k for k in gold if k.endswith("/kind")):
        name = key[:-len("/kind")]
        yield (name, str(gold[key]), gold[f"{name}/in"], tuple(int(v) for v in gold[f"{name}/factor"]), str(gold[f"{name}/raises"]),
               str(gold[f"{name}/raises_floor"]), gold.get(f"{name}/out"))


def oracle_call(kind, arr, factor):
    return DO.downsample_with_averaging(arr, factor) if kind == "average" else DO.downsample_segmentation(arr, factor)


def exhaustive_3d(dtype):
    """Every 2x2x2 block over {0, 1, 2, 3, max}: 390,625 blocks side by side along x."""
    alphabet = np.array([0, 1, 2, 3, np.iinfo(dtype).max], dtype)
    v = alphabet[np.array(list(itertools.product(range(5), repeat=8)), np.int8)]
    a = np.zeros((2, 2, 2 * len(v)), dtype)
    for i in range(8):
        a[i >> 2, (i >> 1) & 1, (i & 1)::2] = v[:, i]
    return a


def exhaustive_2d(dtype, preserved):
    """Every 2x2 block over {0, 1, 2, 3, max} (625), in the plane of the two axes other than ``preserved``."""
    alphabet = np.array([0, 1, 2, 3, np.iinfo(dtype).max], dtype)
    v = alphabet[np.array(list(itertools.product(range(5), repeat=4)), np.int8)]   # a, b, c, d
    plane = np.zeros((2, 2 * len(v)), dtype)
    for i in range(4):
        plane[i >> 1, (i & 1)::2] = v[:, i]
    a = np.stack([plane, plane[::-1]])          # the preserved axis holds two different planes
    return np.moveaxis(a, 0, preserved).copy()


# ------------------------------------------------------------------------------------------------------------
# the oracle against the real reference
# ------------------------------------------------------------------------------------------------------------
def test_golden_covers_the_issue_cases(gold):
    cases = list(golden_cases(gold))
    avg = {f for _, k, _, f, *_ in cases if k == "average"}
    assert avg == {(1, 1, 1), (2, 2, 2), (1, 2, 2), (3, 2, 5), (4, 4, 4)}
    seg = [(a.dtype, a.shape, f) for _, k, a, f, *_ in cases if k == "segmentation"]
    assert {d.name for d, _, _ in seg} == {"uint32", "uint64", "int64", "bool"}
    assert {f for *_, f in seg} >= {(2, 2, 2), (1, 2, 2), (2, 2, 1), (2, 1, 2), (4, 4, 4), (1, 4, 4), (3, 3, 1)}
    assert any(all(s % 2 == 0 for s in shape) for _, shape, _ in seg) and any(all(s % 2 for s in shape) for _, shape, _ in seg)
    # multi-level factors raise in the unmodified module and run with factor // 2; some raise either way
    assert any(r == "TypeError" and not rf for *_, r, rf, _ in cases)
    assert any(r and rf for *_, r, rf, _ in cases)
    assert any(n.startswith("wrap_") for n, *_ in cases)


def test_oracle_against_golden(gold):
    for name, kind, arr, factor, raises, raises_floor, want in golden_cases(gold):
        if raises and raises_floor:
            with pytest.raises(ValueError):
                oracle_call(kind, arr, factor)
            continue
        out = oracle_call(kind, arr, factor)
        assert out.dtype == want.dtype, name
        np.testing.assert_array_equal(out, want, err_msg=name)


def _live(fn):
    from oracle import downsample_harness as DH
    if not DH.available():
        pytest.skip("the reference tree is not available here (the golden vectors pin the oracle everywhere)")
    return fn(DH)


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
def test_oracle_exhaustive_2x2x2_against_live_reference(dtype):
    a = exhaustive_3d(dtype)
    want = _live(lambda DH: DH.segmentation(a, (2, 2, 2)))
    np.testing.assert_array_equal(DO.downsample_segmentation(a, (2, 2, 2)), want)


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
@pytest.mark.parametrize("preserved", [0, 1, 2])
def test_oracle_exhaustive_2x2_against_live_reference(dtype, preserved):
    a = exhaustive_2d(dtype, preserved)
    factor = tuple(1 if i == preserved else 2 for i in range(3))
    want = _live(lambda DH: DH.segmentation(a, factor))
    np.testing.assert_array_equal(DO.downsample_segmentation(a, factor), want)


def random_case(seed):
    rng = np.random.default_rng(900 + seed)
    shape = tuple(int(v) for v in rng.integers(1, 6, 3) * 2 + rng.integers(0, 2, 3) * (seed % 2))
    dtype = (np.uint32, np.uint64, np.int64, bool, np.uint8)[seed % 5]
    if dtype == bool:
        a = rng.random(shape) < 0.5
    elif dtype == np.uint8:
        a = rng.integers(0, 256, shape, dtype=np.uint8)
    else:
        top = np.array(-1).astype(dtype) if np.dtype(dtype).kind == "i" else np.iinfo(dtype).max
        a = np.array([0, 1, 2, top, 5], dtype)[rng.integers(0, 5, shape)]
    factors = [(2, 2, 2), (1, 2, 2), (2, 1, 2), (2, 2, 1), (4, 4, 4), (1, 4, 4), (3, 3, 1), (1, 1, 2), (2, 4, 4), (3, 2, 5)]
    return a, factors


@pytest.mark.parametrize("seed", range(20))
def test_oracle_against_live_reference_on_every_branch(seed):
    """Odd and even shapes; every branch of the dispatch: averaging, striding (bool, no power of two, odd 3-D shape),
    countless2d (odd and even sides), countless3d, multi-level and refused factors."""
    a, factors = random_case(seed)

    def run(DH):
        for f in factors:
            if a.dtype == np.uint8:
                np.testing.assert_array_equal(DO.downsample_with_averaging(a, f), DH.average(a, f), err_msg=str(f))
                continue
            try:
                want = DH.segmentation(a, f, floor_division=True)
            except IndexError:   # its 2x2 path on a 3-D array (a deviation: accepted here)
                continue
            except (TypeError, ValueError):
                with pytest.raises(ValueError):
                    DO.downsample_segmentation(a, f)
                continue
            got = DO.downsample_segmentation(a, f)
            assert got.dtype == want.dtype
            np.testing.assert_array_equal(got, want, err_msg=f"{a.dtype} {a.shape} {f}")
            if not DH.raises(a, f):
                np.testing.assert_array_equal(DH.segmentation(a, f), want)
    _live(run)


def test_oracle_thumbnail_against_golden(gold):
    """`quantize --mode z` and (1,2,2) averagings against the pyramid of the reference's downsample_and_upload."""
    mip = int(gold["thumbnail/mip"])
    assert mip == 5   # max_mip 6 from mip 0 with the first level skipped: five (1,2,2) levels
    np.testing.assert_array_equal(DO.thumbnail(gold["thumbnail/in"], mip)[-1], gold["thumbnail/out"])


def test_oracle_thumbnail_against_live_reference():
    aff = np.random.default_rng(11).random((3, 2, 140, 131), dtype=np.float32)
    mip, want = _live(lambda DH: DH.thumbnail(aff))
    np.testing.assert_array_equal(DO.thumbnail(aff, mip)[-1], want)


def test_command_dispatch():
    with pytest.raises(TypeError, match="only support image or segmentation"):
        DO.downsample(np.zeros((2, 2, 2), np.float32))
    with pytest.raises(TypeError):
        DO.downsample(np.zeros((3, 2, 2, 2), np.uint32))
    assert DO.downsample(np.zeros((4, 4, 4), np.uint8)).shape == (2, 2, 2)
    assert DO.downsample(np.zeros((4, 4, 4), bool)).dtype == bool
    with pytest.raises(ValueError):
        DO.downsample_with_averaging(np.zeros((2, 2, 2), np.uint8), (41, 41, 40))   # 67240 voxels > 65793


# ------------------------------------------------------------------------------------------------------------
# the device code on the host (one-lane CUDA shim)
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("downsample", tmp_path_factory)
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    lib.emu_average.argtypes = [vp, i64, i64, i64, C.POINTER(i64 * 3), vp]
    lib.emu_plan.argtypes = [C.c_int, i64, i64, i64, i64, i64, i64, vp]
    lib.cfb_downsample_workspace.argtypes = [i32, i64, i64, i64, C.POINTER(i64 * 3), C.POINTER(i64 * 3), C.POINTER(i64)]
    lib.cfb_downsample_segmentation_device.argtypes = [vp, i32, i64, i64, i64, C.POINTER(i64 * 3), vp, vp, vp]
    return lib


def emu_average(lib, arr, factor, out):
    """cfb_downsample_average_device -> 1 when it ran the vectorised kernel, 0 for the generic one."""
    path = lib.emu_average(C.c_void_p(arr.ctypes.data), *arr.shape, C.byref((C.c_int64 * 3)(*factor)), C.c_void_p(out.ctypes.data))
    assert path >= 0, lib.cfb_last_error()
    return path


def emu_run(lib, arr, factor):
    """-> the emulated kernels' result, or None when the plan refuses the factor."""
    arr = np.ascontiguousarray(arr)
    p = lambda a: C.c_void_p(a.ctypes.data)
    if arr.dtype == np.uint8:
        out = np.zeros(tuple(-(-s // f) for s, f in zip(arr.shape, factor)), np.uint8)
        emu_average(lib, arr, factor, out)
        return out
    plan = np.zeros(5 * 64, np.int64)
    n = lib.emu_plan(KINDS[arr.dtype], *arr.shape, *factor, p(plan))
    if n < 0:
        return None
    shape = tuple(plan[5 * n - 3: 5 * n]) if n else arr.shape
    out = np.zeros(shape, arr.dtype)
    src = arr.copy()
    from chunkflow_b200._native import DTYPE_BOOL, DTYPE_U32, DTYPE_U64
    dtype = (DTYPE_BOOL, DTYPE_U32, DTYPE_U64)[KINDS[arr.dtype]]
    f, work = (C.c_int64 * 3)(*factor), C.c_int64()
    assert lib.cfb_downsample_workspace(dtype, *arr.shape, C.byref(f), None, C.byref(work)) == 0, lib.cfb_last_error()
    ws = np.zeros(max(work.value, 1), np.uint8)
    assert lib.cfb_downsample_segmentation_device(p(src), dtype, *arr.shape, C.byref(f), p(ws), p(out), None) == 0, lib.cfb_last_error()
    np.testing.assert_array_equal(src, arr)   # the input is only read
    return out


def assert_emulation_matches_oracle(lib, arr, factor):
    try:
        want = oracle_call("average" if arr.dtype == np.uint8 else "segmentation", arr, factor)
    except ValueError:
        assert emu_run(lib, arr, factor) is None, factor
        return
    a = arr.view(np.uint64) if arr.dtype == np.int64 else arr
    got = emu_run(lib, a, factor)
    assert got is not None, factor
    np.testing.assert_array_equal(got.view(arr.dtype) if arr.dtype == np.int64 else got, want, err_msg=f"{arr.dtype} {factor}")


def test_emulation_plan_matches_oracle(emu):
    p = lambda a: C.c_void_p(a.ctypes.data)
    for dtype, shape, factor in itertools.product((np.uint32, bool), ((8, 8, 8), (5, 6, 7), (4, 7, 8), (16, 2, 3)),
                                                  itertools.product((1, 2, 3, 4, 8), repeat=3)):
        plan = np.zeros(5 * 64, np.int64)
        n = emu.emu_plan(KINDS[np.dtype(dtype)], *shape, *factor, p(plan))
        try:
            want = DO.plan(dtype, shape, factor)
        except ValueError:
            assert n == -1, (dtype, shape, factor)
            continue
        algos = {DO.STRIDE: 0, DO.COUNTLESS2D: 1, DO.COUNTLESS3D: 2}
        assert n == len(want), (dtype, shape, factor)
        for i, (algo, _, preserved, out) in enumerate(want):
            assert tuple(plan[5 * i: 5 * i + 5]) == (algos[algo], -1 if preserved is None else preserved) + out


def test_emulation_against_golden(emu, gold):
    for name, kind, arr, factor, raises, raises_floor, want in golden_cases(gold):
        if raises and raises_floor:
            assert emu_run(emu, arr.view(np.uint64) if arr.dtype == np.int64 else arr, factor) is None, name
            continue
        assert_emulation_matches_oracle(emu, arr, factor)


def aligned(shape, dtype, offset=0):
    """A C-order array of ``shape`` that starts ``offset`` bytes after a 16-byte boundary."""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    buf = np.zeros(n + 32, np.uint8)
    start = (-buf.ctypes.data) % 16 + offset
    return buf[start:start + n].view(dtype).reshape(shape)


@pytest.mark.parametrize("factor", [(1, 2, 2), (2, 2, 2), (2, 2, 4), (1, 1, 2)])
@pytest.mark.parametrize("shape", [(5, 7, 48), (4, 6, 32), (1, 1, 16), (3, 9, 50)])
@pytest.mark.parametrize("offset", [0, 1])
def test_emulation_average_both_paths(emu, factor, shape, offset):
    """The vectorised kernel for (1,2,2) and (2,2,2) on 16-byte aligned rows (odd z / y edges clipped), the generic one for
    other factors, rows of no multiple of 16 bytes and unaligned starts."""
    rng = np.random.default_rng(sum(shape) + offset)
    a = aligned(shape, np.uint8, offset)
    a[...] = rng.integers(0, 256, shape, dtype=np.uint8)
    a[0, 0, :8] = 255
    o = tuple(-(-s // k) for s, k in zip(shape, factor))
    out = aligned(o, np.uint8)
    path = emu_average(emu, a, factor, out)
    assert path == (factor[1:] == (2, 2) and factor[0] <= 2 and shape[2] % 16 == 0 and offset == 0)
    np.testing.assert_array_equal(out, DO.downsample_with_averaging(a, factor))


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
def test_emulation_exhaustive_2x2x2(emu, dtype):
    a = exhaustive_3d(dtype)
    np.testing.assert_array_equal(emu_run(emu, a, (2, 2, 2)), DO.downsample_segmentation(a, (2, 2, 2)))


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
@pytest.mark.parametrize("preserved", [0, 1, 2])
def test_emulation_exhaustive_2x2(emu, dtype, preserved):
    a = exhaustive_2d(dtype, preserved)
    factor = tuple(1 if i == preserved else 2 for i in range(3))
    np.testing.assert_array_equal(emu_run(emu, a, factor), DO.downsample_segmentation(a, factor))


@pytest.mark.parametrize("seed", range(20))
def test_emulation_random_shapes_every_branch(emu, seed):
    a, factors = random_case(seed)
    for f in factors:
        assert_emulation_matches_oracle(emu, a, f)


# ------------------------------------------------------------------------------------------------------------
# command line and wrappers, without a device
# ------------------------------------------------------------------------------------------------------------
def test_downsample_options_are_spelled_like_the_reference():
    from chunkflow_b200.flow.cli import main
    cmd = main.commands["downsample"]
    mine = {o.name: tuple(o.opts) for o in cmd.params}
    assert mine == {"input_chunk_name": ("--input-chunk-name", "-i"), "output_chunk_name": ("--output-chunk-name", "-o"),
                    "factor": ("--factor", "-f")}
    factor = next(o for o in cmd.params if o.name == "factor")
    assert factor.nargs == 3 and tuple(factor.default) == (2, 2, 2)
    from oracle import reference_harness as H
    if not H.available():
        pytest.skip("the reference tree is not available here")
    with open(os.path.join(H.REFERENCE_ROOT, "chunkflow", "flow", "flow.py")) as f:
        text = f.read()
    body = text[text.index("@main.command('downsample')"):]
    body = body[:body.index("@operator")]
    theirs = re.findall(r"@click\.option\('(--[\w-]+)',\s*'(-\w)'", body)
    assert sorted(theirs) == sorted(mine.values())
    assert "nargs=3, default=(2,2,2)" in body


def test_workspace_plan_needs_no_device():
    from chunkflow_b200 import _native
    assert _native.downsample_workspace(_native.DTYPE_U32, (8, 8, 8), (2, 2, 2)) == ((4, 4, 4), 0)
    assert _native.downsample_workspace(_native.DTYPE_U64, (8, 8, 8), (4, 4, 4)) == ((2, 2, 2), 512)
    assert _native.downsample_workspace(_native.DTYPE_U32, (5, 7, 9), (1, 2, 2)) == ((5, 4, 5), 0)
    assert _native.downsample_workspace(_native.DTYPE_BOOL, (5, 7, 9), (4, 4, 4)) == ((2, 2, 3), 0)
    with pytest.raises(ValueError, match="factor of 0"):
        _native.downsample_workspace(_native.DTYPE_U32, (8, 8, 8), (1, 1, 2))
    with pytest.raises(ValueError, match="factor of 0"):
        _native.downsample_workspace(_native.DTYPE_U64, (8, 8, 8), (2, 2, 4))
    assert _native.downsample_workspace(_native.DTYPE_U64, (7, 8, 8), (2, 2, 4))[0] == (4, 4, 2)   # odd: one strided level


@pytest.mark.skipif(has_gpu(), reason="checks the no-GPU failure mode")
def test_entry_points_raise_without_a_gpu():
    from chunkflow_b200 import _native
    with pytest.raises(_native.NativeError) as ei:
        _native.downsample_average_device(1 << 20, (4, 4, 4), (2, 2, 2), 1 << 24)
    assert ei.value.code == _native.ERR_CUDA
    with pytest.raises(_native.NativeError) as ei:
        _native.downsample_segmentation_device(1 << 20, _native.DTYPE_U32, (4, 4, 4), (2, 2, 2), 0, 1 << 24)
    assert ei.value.code == _native.ERR_CUDA


def test_wrappers_validate_before_the_library_is_touched(monkeypatch):
    from chunkflow_b200 import _native
    monkeypatch.setattr(_native, "load", lambda: pytest.fail("the native library must not be reached"))
    with pytest.raises(ValueError, match="less than one"):
        _native.downsample_average_device(16, (4, 4, 4), (0, 2, 2), 32)
    with pytest.raises(ValueError):
        _native.downsample_average_device(16, (4, 0, 4), (2, 2, 2), 32)
    with pytest.raises(ValueError):
        _native.downsample_workspace(_native.DTYPE_U32, (4, 4, 4), (2, 2))
    with pytest.raises(TypeError):
        _native.downsample_workspace(_native.DTYPE_U8, (4, 4, 4), (2, 2, 2))
    with pytest.raises(TypeError):
        _native.downsample_segmentation_device(16, _native.DTYPE_F32, (4, 4, 4), (2, 2, 2), 0, 32)
    with pytest.raises(ValueError, match="less than one"):
        _native.downsample_segmentation_device(16, _native.DTYPE_U64, (4, 4, 4), (2, -2, 2), 0, 32)


def test_native_refusals_are_value_errors():
    from chunkflow_b200 import _native
    with pytest.raises(ValueError, match="65793"):
        _native.downsample_average_device(1 << 20, (4, 4, 4), (41, 41, 40), 1 << 24)
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        _native.downsample_workspace(_native.DTYPE_U32, (4, 4, 4), (2 ** 16, 2 ** 16, 1))
