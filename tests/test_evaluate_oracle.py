"""`evaluate-segmentation` (DESIGN.md section 0, row f5; reference chunk/segmentation.py:33-67 -> lib/gala/evaluate.py) on the CPU:
the numpy oracle (oracle/evaluation_oracle.py) against golden vectors of the REAL reference
(tests/golden/evaluate_reference.npz, made by tests/golden/make_golden_evaluate.py) and, where the reference tree exists,
against the live reference; csrc/evaluate.cu and its host scoring code (csrc/evaluate_scores.h), compiled for the host behind a
one-lane CUDA shim (tests/host_emulation), against the oracle."""
import ctypes as C
import io
import os
import warnings
from contextlib import redirect_stdout

import numpy as np
import pytest

import host_emulation
from oracle import evaluation_oracle as EV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "evaluate_reference.npz")
SCORE_NAMES = ("rand_index", "adjusted_rand_index", "variation_of_information", "fowlkes_mallows_index")


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def golden_cases(gold):
    return sorted({k.split("/")[0] for k in gold})


def assert_scores_match(got: dict, row, vi_tol=1e-12):
    """row: (threshold, RI, ARI, VI, FM, false merges, false splits) of the reference.  RI, ARI, FM and the edit distance
    bit-exact (NaN where the reference has NaN), VI within vi_tol."""
    _, ri, ari, vi, fm, merges, splits = row
    for name, want in (("rand_index", ri), ("adjusted_rand_index", ari), ("fowlkes_mallows_index", fm)):
        g = float(got[name])
        assert (np.isnan(g) and np.isnan(want)) or g == want, (name, g, want)
    g = float(got["variation_of_information"])
    assert (np.isnan(g) and np.isnan(vi)) or abs(g - vi) <= vi_tol, ("variation_of_information", g, vi)
    assert tuple(float(v) for v in got["edit_distance"]) == (merges, splits)


# ------------------------------------------------------------------------------------------------------------
# the oracle against the real reference
# ------------------------------------------------------------------------------------------------------------
def test_golden_covers_the_issue_cases(gold):
    names = golden_cases(gold)
    assert {"all_zero", "one_label", "all_distinct", "blobs_int64", "random_u32"} <= set(names)
    assert {gold[f"{n}/seg"].dtype.name for n in names} >= {"uint32", "uint64", "int64"}


def test_oracle_against_golden(gold):
    for name in golden_cases(gold):
        seg, gt = gold[f"{name}/seg"], gold[f"{name}/gt"]
        s, g, c = EV.contingency_triples(seg, gt)
        np.testing.assert_array_equal(np.stack([s, g, c], 1), gold[f"{name}/table"], err_msg=name)
        for row in gold[f"{name}/scores"]:
            assert_scores_match(EV.evaluate(seg, gt, size_threshold=row[0]), row)


def test_degenerate_cases_are_nan_like_the_reference(gold):
    nan = float("nan")
    want = {"all_zero": (1.0, nan, nan, 1.0, (0.0, 0.0)), "one_label": (1.0, nan, 0.0, 1.0, (-1.0, 0.0))}
    for name, (ri, ari, vi, fm, ed) in want.items():
        r = EV.evaluate(gold[f"{name}/seg"], gold[f"{name}/gt"], 1000)
        np.testing.assert_equal([r["rand_index"], r["adjusted_rand_index"], r["variation_of_information"], r["fowlkes_mallows_index"]],
                                [ri, ari, vi, fm])
        assert r["edit_distance"] == ed
    r = EV.evaluate(gold["all_distinct/seg"], gold["all_distinct/gt"], 0)
    np.testing.assert_equal([r["rand_index"], r["adjusted_rand_index"], r["variation_of_information"], r["fowlkes_mallows_index"]],
                            [1.0, nan, 0.0, nan])
    assert r["edit_distance"] == (0.0, 0.0)


def test_printed_lines_match_the_reference(gold):
    from chunkflow_b200.chunk.segmentation import report
    for name in golden_cases(gold):
        for row, printed in zip(gold[f"{name}/scores"], gold[f"{name}/printed"]):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                assert report(EV.evaluate(gold[f"{name}/seg"], gold[f"{name}/gt"], row[0])) == str(printed), name


def _live_case(seed):
    rng = np.random.default_rng(1000 + seed)
    shape = tuple(int(v) for v in rng.integers(2, 14, 3))
    kind = seed % 3
    if kind == 0:      # random labels, 0 included
        seg = rng.integers(0, int(rng.integers(1, 30)), shape)
        gt = rng.integers(0, int(rng.integers(1, 30)), shape)
    elif kind == 1:    # a copy of the segmentation with a few voxels changed
        seg = rng.integers(0, 6, shape)
        gt = seg.copy()
        m = rng.random(shape) < 0.1
        gt[m] = rng.integers(0, 9, int(m.sum()))
    else:              # no zeros, ids up to 2^22
        seg = rng.integers(1, 2 ** 22, 4)[rng.integers(0, 4, shape)]
        gt = rng.integers(1, 2 ** 22, 5)[rng.integers(0, 5, shape)]
    dtype = (np.uint32, np.int64, np.uint64)[seed % 3]
    return seg.astype(dtype), gt.astype(dtype), float((0, 1, 3, 10, 1000)[seed % 5])


@pytest.mark.parametrize("seed", range(30))
def test_oracle_against_live_reference(seed):
    from oracle import evaluation_harness as EH
    if not EH.available():
        pytest.skip("the reference tree is not available here (the golden vectors pin the oracle everywhere)")
    Segmentation, Chunk, _ = EH.import_reference_evaluation()
    seg, gt, thr = _live_case(seed)
    with warnings.catch_warnings(), redirect_stdout(io.StringIO()):
        warnings.simplefilter("ignore")
        r = Segmentation(Chunk(seg.copy())).evaluate(Chunk(gt.copy()), size_threshold=thr)
        mine = EV.evaluate(seg, gt, thr)
    row = (thr, r["rand_index"], r["adjusted_rand_index"], r["variation_of_information"], r["fowlkes_mallows_index"],
           *r["edit_distance"])
    assert_scores_match(mine, np.array(row, np.float64))


def test_oracle_is_invariant_under_relabelling_with_wide_ids():
    rng = np.random.default_rng(5)
    seg, gt = rng.integers(0, 7, (5, 6, 7)), rng.integers(0, 5, (5, 6, 7))
    base = EV.evaluate(seg, gt, 2)
    wide = np.array([0, 2 ** 63 + 3, 2 ** 64 - 1, 2 ** 40, 1, 2 ** 63, 99], np.uint64)   # 0 -> 0 keeps the ignored label
    r = EV.evaluate(wide[seg], wide[gt], 2)
    for k in SCORE_NAMES:
        np.testing.assert_equal(r[k], base[k])
    assert r["edit_distance"] == base["edit_distance"]


# ------------------------------------------------------------------------------------------------------------
# the device code on the host (one-thread CUDA shim)
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("evaluate", tmp_path_factory)
    from chunkflow_b200._native import SegScores
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    lib.cfb_evaluate_workspace.argtypes = [i64]
    lib.cfb_evaluate_workspace.restype = i64
    lib.cfb_contingency_device.argtypes = [vp, i32, vp, i32, i64, i64, i64, vp, i64, C.POINTER(i64), vp]
    lib.cfb_contingency_scores.argtypes = [vp, i64, C.c_double, C.POINTER(SegScores), vp]   # refuses another struct_size
    lib.cfb_contingency_read.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    return lib


def emu_evaluate(lib, seg, gt, size_threshold, slots=None):
    from chunkflow_b200._native import SegScores
    seg, gt = np.ascontiguousarray(seg), np.ascontiguousarray(gt)
    assert seg.dtype.itemsize in (1, 4, 8) and gt.dtype.itemsize in (1, 4, 8)
    if slots is None:
        slots = 32
        while slots < 4 * seg.size:
            slots <<= 1
    from chunkflow_b200._native import DTYPE_U8, DTYPE_U32, DTYPE_U64, ERR_CAPACITY
    dtype = {1: DTYPE_U8, 4: DTYPE_U32, 8: DTYPE_U64}
    s, g, c = np.empty(slots, np.uint64), np.empty(slots, np.uint64), np.empty(slots, np.uint32)
    out = SegScores(struct_size=C.sizeof(SegScores))
    p = lambda a: C.c_void_p(a.ctypes.data)
    work = np.zeros(lib.cfb_evaluate_workspace(slots) // 8, np.uint64)
    n = C.c_int64()
    rc = lib.cfb_contingency_device(p(seg), dtype[seg.dtype.itemsize], p(gt), dtype[gt.dtype.itemsize], 1, 1, seg.size, p(work), slots,
                                    C.byref(n), None)
    if rc == ERR_CAPACITY:
        return -1, None, None
    assert rc == 0, lib.cfb_last_error()
    assert lib.cfb_contingency_scores(p(work), slots, size_threshold, C.byref(out), None) == 0, lib.cfb_last_error()
    n = n.value
    assert lib.cfb_contingency_read(p(work), slots, n, p(s), p(g), p(c), None) == 0, lib.cfb_last_error()
    return n, (s[:n], g[:n], c[:n]), out.as_dict()


def assert_emulation_matches_oracle(lib, seg, gt, thr):
    n, (s, g, c), st = emu_evaluate(lib, seg, gt, thr)
    os_, og, oc = EV.contingency_triples(seg, gt)
    np.testing.assert_array_equal(s, os_); np.testing.assert_array_equal(g, og); np.testing.assert_array_equal(c, oc)
    want = EV.statistics(os_, og, oc, thr)
    for k, v in want.items():
        if k.startswith("xlog"):
            assert st[k] == pytest.approx(v, rel=1e-14, abs=1e-9), k
        else:
            assert st[k] == v, k
    return st


def test_emulation_against_golden(emu, gold):
    for name in golden_cases(gold):
        seg, gt = gold[f"{name}/seg"], gold[f"{name}/gt"]
        for row in gold[f"{name}/scores"]:
            st = assert_emulation_matches_oracle(emu, seg.astype(np.uint64) if seg.dtype.kind == "i" else seg,
                                                 gt.astype(np.uint64) if gt.dtype.kind == "i" else gt, row[0])
            assert_scores_match(dict(st, edit_distance=(st["false_merges"], st["false_splits"])), row)


@pytest.mark.parametrize("seed", range(6))
def test_emulation_against_oracle_mixed_dtypes_and_wide_ids(emu, seed):
    rng = np.random.default_rng(seed)
    shape = (4, 9, 11)
    pool = np.array([0, 1, 2, 2 ** 63 + seed, 2 ** 64 - 1, 2 ** 32, 255, 77], np.uint64)
    seg = pool[rng.integers(0, pool.size, shape)]
    gt8 = rng.integers(0, 4, shape).astype(np.uint8)
    gt32 = rng.integers(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    assert_emulation_matches_oracle(emu, seg, gt8, 3)
    assert_emulation_matches_oracle(emu, gt32, seg, 0)
    assert_emulation_matches_oracle(emu, gt8, gt32, 1000)


def test_emulation_reports_a_full_table(emu):
    seg = np.arange(200, dtype=np.uint32).reshape(2, 10, 10)
    n, _, _ = emu_evaluate(emu, seg, seg, 0, slots=64)
    assert n == -1
