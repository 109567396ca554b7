"""Segmentation clean-up (DESIGN.md section 0, row f6; reference chunk/segmentation.py:69-109, flow/flow.py:2015-2050) on the CPU:
the numpy oracle (oracle/relabel_oracle.py) against golden vectors of the REAL reference's methods
(tests/golden/relabel_reference.npz, made by tests/golden/make_golden_relabel.py) and, where the reference tree exists, against
the live reference; csrc/relabel.cu, compiled for the host behind a one-lane CUDA shim (tests/host_emulation), against the oracle; the command's option names; the wrappers' argument checks."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import host_emulation
from oracle import relabel_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "relabel_reference.npz")


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def golden_calls(gold):
    """(case, input array, method, argument, resulting array, returned value or None, printed text) of every recorded call."""
    for key in sorted(k for k in gold if k.endswith("/method")):
        name, k, _ = key.split("/")
        arg = gold[f"{name}/{k}/arg"]
        if arg.dtype.kind == "U":
            arg = None if str(arg) == "None" else str(arg)
        elif arg.ndim == 0:
            arg = int(arg)
        ret = gold[f"{name}/{k}/ret"]
        yield (name, gold[f"{name}/in"], str(gold[key]), arg, gold[f"{name}/{k}/out"], None if ret.dtype == np.int64 else int(ret),
               str(gold[f"{name}/{k}/printed"]))


def oracle_call(arr, method, arg):
    """-> (array, returned value, printed text) like the reference's method."""
    if method == "mask_fragments":
        out, text = RO.mask_fragments(arr, arg)
        return out, None, text
    if method == "mask_except":
        out, text = RO.mask_except(arr, arg)
        return out, None, text
    out, new_base = RO.remap(arr, arg)
    return out, new_base, ""


# ------------------------------------------------------------------------------------------------------------
# the oracle against the real reference
# ------------------------------------------------------------------------------------------------------------
def test_golden_covers_the_issue_cases(gold):
    calls = list(golden_calls(gold))
    assert {c[1].dtype.name for c in calls} >= {"uint8", "uint32", "uint64", "int64"}
    assert any(not (c[1] == 0).any() for c in calls) and any((c[1] == 0).any() for c in calls)
    # a count exactly equal to the threshold; keep ids that do not occur; the all-zero chunk with base_id > 0
    assert any(m == "mask_fragments" and (np.unique(a, return_counts=True)[1] == arg).any() for _, a, m, arg, *_ in calls)
    assert any(m == "mask_except" and arg is not None and not isinstance(arg, str) and not np.isin(arg, a).all()
               for _, a, m, arg, *_ in calls)
    assert any(n == "all_zero" and m == "remap" and arg > 0 and ret == 0 for n, _, m, arg, _, ret, _ in calls)
    assert any("masking out" in c[6] for c in calls) and any("we have not selected" in c[6] for c in calls)


def test_oracle_against_golden(gold):
    for name, arr, method, arg, want, ret, printed in golden_calls(gold):
        out, r, text = oracle_call(arr, method, arg)
        assert out.dtype == want.dtype, (name, method)
        np.testing.assert_array_equal(out, want, err_msg=f"{name} {method} {arg}")
        assert r == ret and text == printed, (name, method, arg)


def _live_case(seed):
    rng = np.random.default_rng(500 + seed)
    shape = tuple(int(v) for v in rng.integers(2, 12, 3))
    dtype = (np.uint8, np.uint32, np.uint64, np.int64)[seed % 4]
    pool = rng.integers(0 if seed % 3 else 1, 250, int(rng.integers(1, 25)))
    arr = pool[rng.integers(0, pool.size, shape)]
    if seed % 2:
        arr[:, :, : shape[2] // 2] = arr[:, :, :1]
    return arr.astype(dtype), rng


@pytest.mark.parametrize("seed", range(24))
def test_oracle_against_live_reference(seed):
    from oracle import relabel_harness as RH
    if not RH.available():
        pytest.skip("the reference tree is not available here (the golden vectors pin the oracle everywhere)")
    arr, rng = _live_case(seed)
    ids = np.unique(arr)
    keep = set(int(i) for i in rng.choice(ids, size=max(1, ids.size // 2), replace=False)) | {251}
    for method, arg in (("mask_fragments", int(rng.integers(0, 12))), ("mask_except", keep),
                        ("mask_except", ",".join(str(i) for i in sorted(keep))), ("remap", int(rng.integers(0, 3)) * 1000)):
        want, ret, printed = RH.run(method, arr, arg)
        out, r, text = oracle_call(arr, method, arg)
        assert out.dtype == want.dtype
        np.testing.assert_array_equal(out, want, err_msg=f"{method} {arg}")
        assert (None if ret is None else int(ret)) == r and text == printed


def test_mask_out_objects_is_dust_then_keep_list():
    rng = np.random.default_rng(3)
    arr = rng.integers(0, 40, (5, 8, 9)).astype(np.uint32)
    arr[:, :4] = 7
    out, text = RO.mask_out_objects(arr, 8, "7,3,4,5,6")
    step, line = RO.mask_fragments(arr, 8)
    np.testing.assert_array_equal(out, RO.mask_except(step, [7, 3, 4, 5, 6])[0])
    assert text == line and set(np.unique(out)) <= {0, 3, 4, 5, 6, 7}


def test_selected_ids_parsing(tmp_path, capsys):
    from chunkflow_b200.chunk.device import selected_ids
    assert selected_ids(None) is None
    np.testing.assert_array_equal(np.sort(selected_ids("34,45,56,34")), np.array([34, 45, 56], np.uint64))
    np.testing.assert_array_equal(selected_ids([2 ** 64 - 1, -1]), np.array([2 ** 64 - 1, 2 ** 64 - 1], np.uint64))
    np.testing.assert_array_equal(selected_ids(np.array([5, 2 ** 63 + 5], np.uint64)), np.array([5, 2 ** 63 + 5], np.uint64))
    assert selected_ids([]).size == 0 and selected_ids(set()).dtype == np.uint64
    path = tmp_path / "ids.json"
    path.write_text(json.dumps([3, 4, 4, 9]))
    np.testing.assert_array_equal(np.sort(selected_ids(str(path))), np.array([3, 4, 9], np.uint64))
    assert capsys.readouterr().out == "number of selected objects: 3\n"
    (tmp_path / "empty.json").write_text("[]")
    with pytest.raises(AssertionError):
        selected_ids(str(tmp_path / "empty.json"))
    with pytest.raises(ValueError, match="local json"):
        selected_ids("gs://bucket/ids.json")
    with pytest.raises(ValueError):
        selected_ids([2 ** 64])
    with pytest.raises(ValueError):
        selected_ids("3,,4")


# ------------------------------------------------------------------------------------------------------------
# the device code on the host (one-lane CUDA shim)
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("relabel", tmp_path_factory)
    i32, i64, vp, pi64 = C.c_int32, C.c_int64, C.c_void_p, C.POINTER(C.c_int64)
    lib.cfb_label_table_workspace.argtypes = [i64, i64]
    lib.cfb_label_table_workspace.restype = i64
    lib.cfb_label_table_device.argtypes = [vp, i32, i64, i64, i64, vp, i64, pi64, vp]
    lib.cfb_label_table_read.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    lib.cfb_label_table_plan.argtypes = [vp, i64, i64, i32, i64, vp, i64, i32, C.c_uint64, pi64, pi64, C.POINTER(C.c_uint64), vp]
    lib.cfb_label_apply_device.argtypes = [vp, i32, i64, vp, i64, vp, i32, vp]
    return lib


def aligned_copy(arr):
    """A copy of ``arr`` that starts on a 16-byte boundary, as the library requires."""
    buf = np.zeros(arr.nbytes + 16, np.uint8)
    start = (-buf.ctypes.data) % 16
    out = buf[start:start + arr.nbytes].view(arr.dtype).reshape(arr.shape)
    out[...] = arr
    return out


def emu_relabel(lib, arr, dust=None, keep=None, renumber=False, base_id=0, slots=None, in_place=False):
    """-> (labels, (ids, counts, first), result array, (dust entries, survivors, new maximum)); labels < 0 on failure."""
    arr = np.ascontiguousarray(arr)
    assert arr.dtype in (np.uint8, np.uint32, np.uint64)
    if slots is None:
        slots = 32
        while slots < 4 * arr.size:
            slots <<= 1
    from chunkflow_b200._native import DTYPE_U8, DTYPE_U32, DTYPE_U64, ERR_CAPACITY
    dtype = {1: DTYPE_U8, 4: DTYPE_U32, 8: DTYPE_U64}[arr.dtype.itemsize]
    ids, counts, first = np.empty(slots, np.uint64), np.empty(slots, np.uint32), np.empty(slots, np.uint32)
    src = aligned_copy(arr)
    out = src if in_place else aligned_copy(np.zeros(arr.shape, np.uint64 if renumber else arr.dtype))
    keep_arr = None if keep is None else np.ascontiguousarray(keep, np.uint64)
    p = lambda a: C.c_void_p(a.ctypes.data)
    work = np.zeros(-(-lib.cfb_label_table_workspace(arr.size, slots) // 8), np.uint64)
    n, dust_n, survivors, new_max = C.c_int64(), C.c_int64(), C.c_int64(), C.c_uint64()
    rc = lib.cfb_label_table_device(p(src), dtype, 1, 1, arr.size, p(work), slots, C.byref(n), None)
    if rc == ERR_CAPACITY:
        return -1, None, None, None
    assert rc == 0, lib.cfb_last_error()
    n = n.value
    assert lib.cfb_label_table_read(p(work), slots, n, p(ids), p(counts), p(first), None) == 0, lib.cfb_last_error()
    assert lib.cfb_label_table_plan(p(work), slots, arr.size, int(dust is not None), dust or 0,
                                    p(keep_arr) if keep_arr is not None and keep_arr.size else None,
                                    -1 if keep_arr is None else keep_arr.size, int(renumber), base_id, C.byref(dust_n),
                                    C.byref(survivors), C.byref(new_max), None) == 0, lib.cfb_last_error()
    assert lib.cfb_label_apply_device(p(src), dtype, arr.size, p(work), slots, p(out), DTYPE_U64 if renumber else dtype,
                                      None) == 0, lib.cfb_last_error()
    info = (dust_n.value, survivors.value, new_max.value)
    if not in_place:
        np.testing.assert_array_equal(src, arr)   # the input is only read
    return int(n), (ids[:n], counts[:n], first[:n]), out, tuple(int(v) for v in info)


def assert_emulation_matches_oracle(lib, arr, dust=None, keep=None, base_id=None):
    n, (ids, counts, first), out, info = emu_relabel(lib, arr, dust, keep, base_id is not None, base_id or 0)
    o_ids, o_first, o_counts = RO.unique(arr, return_index=True, return_counts=True)
    np.testing.assert_array_equal(ids, o_ids.astype(np.uint64)); np.testing.assert_array_equal(counts, o_counts)
    np.testing.assert_array_equal(first, o_first)
    want = arr
    if dust is not None:
        want = RO.mask_fragments(want, dust)[0]
        assert info[0] == int((o_counts <= dust).sum())
    if keep is not None:
        want = RO.mask_except_ids(want, keep)
    if base_id is not None:
        want, new_max = RO.remap(want, base_id)
        assert info[2] == new_max
    assert out.dtype == want.dtype
    np.testing.assert_array_equal(out, want)
    assert info[1] == np.unique(want[want != 0]).size
    return out


def test_emulation_against_golden(emu, gold):
    for name, arr, method, arg, want, ret, _ in golden_calls(gold):
        a = arr.astype(np.uint64) if arr.dtype.kind == "i" else arr
        if method == "mask_fragments":
            out = assert_emulation_matches_oracle(emu, a, dust=arg)
        elif method == "mask_except":
            ids, _ = RO.parse_selected_obj_ids(arg)
            if ids is None:
                continue
            out = assert_emulation_matches_oracle(emu, a, keep=RO._ids_u64(ids))
        else:
            out = assert_emulation_matches_oracle(emu, a, base_id=arg)
        np.testing.assert_array_equal(out.astype(want.dtype), want, err_msg=f"{name} {method}")


@pytest.mark.parametrize("seed", range(8))
def test_emulation_wide_ids_mixed_run_lengths_and_combinations(emu, seed):
    rng = np.random.default_rng(seed)
    pool = np.array([0, 1, 2, 2 ** 63 + 5, 2 ** 64 - 1, 2 ** 32, 255, 77, 2 ** 40 + seed], np.uint64)
    n = int(rng.integers(1, 700))                       # sizes that are no multiple of the 2 / 4 / 16 ids of a vector load
    runs = rng.integers(1, (1, 3, 9, 40)[seed % 4] + 1, n)
    wide = np.repeat(pool[rng.integers(0, pool.size, n)], runs)[:n].reshape(1, 1, -1)
    u32 = (wide % np.uint64(2 ** 32)).astype(np.uint32)
    u8 = (wide % np.uint64(7)).astype(np.uint8)
    for arr in (wide, u32, u8):
        ids = np.unique(arr).astype(np.uint64)
        keep = np.concatenate([ids[::2], np.array([12345], np.uint64)])
        assert_emulation_matches_oracle(emu, arr)
        assert_emulation_matches_oracle(emu, arr, dust=int(rng.integers(0, 30)))
        assert_emulation_matches_oracle(emu, arr, keep=keep)
        assert_emulation_matches_oracle(emu, arr, keep=np.zeros(0, np.uint64))
        assert_emulation_matches_oracle(emu, arr, base_id=0)
        assert_emulation_matches_oracle(emu, arr, dust=5, keep=keep, base_id=2 ** 40)


def test_emulation_masks_in_place(emu):
    rng = np.random.default_rng(9)
    arr = np.repeat(rng.integers(0, 9, 90), rng.integers(1, 7, 90)).astype(np.uint32).reshape(1, 1, -1)
    _, _, out, _ = emu_relabel(emu, arr, dust=12, keep=np.arange(1, 6), in_place=True)
    np.testing.assert_array_equal(out, RO.mask_out_objects(arr, 12, [1, 2, 3, 4, 5])[0])


def test_emulation_reports_a_full_table(emu):
    arr = np.arange(200, dtype=np.uint32).reshape(2, 10, 10)
    assert emu_relabel(emu, arr, slots=64)[0] == -1
    assert emu_relabel(emu, arr, slots=1024)[0] == 200


# ------------------------------------------------------------------------------------------------------------
# command line and wrappers, without a device
# ------------------------------------------------------------------------------------------------------------
def _options(cmd):
    return {o.name: tuple(o.opts) for o in cmd.params}


def test_mask_out_objects_options_are_spelled_like_the_reference():
    from chunkflow_b200.flow.cli import main
    mine = _options(main.commands["mask-out-objects"])
    assert mine == {"input_chunk_name": ("--input-chunk-name", "-i"), "output_chunk_name": ("--output_chunk_name", "-o"),
                    "dust_size_threshold": ("--dust-size-threshold", "-d"), "selected_obj_ids": ("--selected-obj-ids", "-s")}
    from oracle import reference_harness as H
    if not H.available():
        pytest.skip("the reference tree is not available here")
    with open(os.path.join(H.REFERENCE_ROOT, "chunkflow", "flow", "flow.py")) as f:
        text = f.read()
    body = text[text.index("@main.command('mask-out-objects')"):]
    body = body[:body.index("@operator")]
    theirs = re.findall(r"@click\.option\('(--[\w-]+)',\s*'(-\w)'", body)
    assert sorted(theirs) == sorted(mine.values())


def test_remap_segmentation_is_marked_as_an_extension():
    from chunkflow_b200.flow.cli import main
    cmd = main.commands["remap-segmentation"]
    assert cmd.help.startswith("(extension)")
    assert _options(cmd)["base_id"] == ("--base-id",)


def test_wrappers_validate_before_the_library_is_touched(monkeypatch):
    from chunkflow_b200 import _native
    monkeypatch.setattr(_native, "load", lambda: pytest.fail("the native library must not be reached"))
    with pytest.raises(ValueError):
        _native.label_table_device(16, _native.DTYPE_U32, (0, 4, 4), 16, 64)
    with pytest.raises(ValueError, match="2\\^32 - 2"):
        _native.label_table_device(16, _native.DTYPE_U32, (2048, 2048, 1024), 16, 64)
    with pytest.raises(TypeError):
        _native.label_table_device(16, _native.DTYPE_F32, (4, 4, 4), 16, 64)
    with pytest.raises(ValueError, match="power of two"):
        _native.label_table_device(16, _native.DTYPE_U32, (4, 4, 4), 16, 48)
    with pytest.raises(ValueError):
        _native.label_table_read(16, 64, 65)
    with pytest.raises(ValueError, match="negative"):
        _native.label_table_plan(16, 64, 64, renumber=True, base_id=-1)
    with pytest.raises(ValueError, match="2\\^64"):
        _native.label_table_plan(16, 64, 64, renumber=True, base_id=2 ** 64)
    with pytest.raises(TypeError):
        _native.label_table_plan(16, 64, 64, renumber=True, base_id=1.5)
    with pytest.raises(ValueError, match="renumber"):
        _native.label_table_plan(16, 64, 64, base_id=5)
    with pytest.raises(TypeError):
        _native.label_table_plan(16, 64, 64, dust_threshold=2.5)
    with pytest.raises(ValueError):
        _native.label_table_plan(16, 64, 64, num_keep=3)
    with pytest.raises(TypeError):
        _native.label_apply_device(16, _native.DTYPE_U64, 64, 16, 64, 32, _native.DTYPE_U32)
    with pytest.raises(ValueError, match="in place"):
        _native.label_apply_device(16, _native.DTYPE_U32, 64, 16, 64, 16, _native.DTYPE_U64)
