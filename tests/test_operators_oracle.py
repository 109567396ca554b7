"""Pins oracle/operators_oracle.py (SURVEY.md section 8 f3) to golden vectors made by the REAL reference
(tests/golden/make_golden_operators.py) and to recorded outputs of the reference classes on seeded random inputs
(tests/golden/operators_reference.npz; `CFB_RECORD_REFERENCE=1` re-records them where the reference tree exists)."""
import io
import os
import warnings
from contextlib import redirect_stderr, redirect_stdout

import numpy as np
import pytest

from oracle import operators_oracle as OP
from oracle import reference_harness as H

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "operators.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


NC_CASES = {"nc_default": dict(), "nc_custom": dict(lower_clip_fraction=0.05, upper_clip_fraction=0.02, minval=0, maxval=200),
            "nc_zero_clip": dict(lower_clip_fraction=0.0, upper_clip_fraction=0.0), "nc_not_per_section": dict(per_section=False)}


@pytest.mark.parametrize("tag", sorted(NC_CASES))
def test_normalize_contrast_golden(gold, tag):
    out = OP.normalize_contrast(gold["image"], **NC_CASES[tag])
    assert out.dtype == np.uint8
    np.testing.assert_array_equal(out, gold[tag])


def test_normalize_contrast_quirks(gold):
    # per_section=False is a no-op in the reference (the whole-array branch is the for loop's else clause)
    np.testing.assert_array_equal(gold["nc_not_per_section"], gold["image"])
    # black and constant sections are left alone by the per-section pass, but the trailing whole-array pass still applies
    assert (gold["nc_default"] != gold["image"]).any()


def test_quantize_maskout_crop_golden(gold):
    np.testing.assert_array_equal(OP.quantize(gold["aff"], "xy"), gold["quant_xy"])
    np.testing.assert_array_equal(OP.quantize(gold["aff"], "z"), gold["quant_z"])
    with pytest.raises(ValueError):
        OP.quantize(gold["aff"], "yz")
    np.testing.assert_array_equal(OP.maskout(gold["mask"], (2, 4, 4), gold["aff"], (1, 1, 1)), gold["maskout_aff"])
    np.testing.assert_array_equal(OP.maskout(gold["mask"], (8, 16, 16), gold["image2"], (4, 4, 4)), gold["maskout_img"])
    a3, o3 = OP.crop_margin(gold["aff"], (5, 6, 7), (1, 2, 3))
    a6, o6 = OP.crop_margin(gold["aff"], (5, 6, 7), (1, 0, 3, 2, 4, 0))
    np.testing.assert_array_equal(a3, gold["crop3"]); assert tuple(o3) == tuple(gold["crop3_offset"])
    np.testing.assert_array_equal(a6, gold["crop6"]); assert tuple(o6) == tuple(gold["crop6_offset"])
    with pytest.raises(ValueError):
        OP.crop_margin(gold["aff"], (0, 0, 0), (1, 2))


RECORDED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "operators_reference.npz")
RECORD = os.environ.get("CFB_RECORD_REFERENCE") == "1"   # re-run the real reference (needs its tree) and rewrite RECORDED


@pytest.fixture(scope="module")
def recorded():
    """Outputs of the real reference classes by key: computed and saved while recording, loaded otherwise."""
    if not RECORD:
        yield dict(np.load(RECORDED))
        return
    if not H.available():
        pytest.fail("CFB_RECORD_REFERENCE=1 needs the reference tree (CHUNKFLOW_REFERENCE_ROOT)")
    H.import_reference()
    warnings.simplefilter("ignore")
    rec = {}
    yield rec
    old = dict(np.load(RECORDED)) if os.path.exists(RECORDED) else {}
    old.update(rec)
    np.savez_compressed(RECORDED, **old)


def _ref(recorded, key, compute):
    if RECORD:
        recorded[key] = np.asarray(compute())
    return recorded[key]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_against_real_reference(recorded, seed):
    def ref_normalize():
        from chunkflow.chunk.image.base import Image
        im = Image(img.copy())
        with redirect_stdout(io.StringIO()), redirect_stderr(io.StringIO()):
            im.normalize_contrast(lo, hi, 1 + seed, 255 - 10 * seed, True)
        return im.array

    def ref_quantize(mode):
        from chunkflow.chunk.affinity_map import AffinityMap
        return AffinityMap(aff.copy()).quantize(mode).array

    def ref_maskout():
        Chunk = H.import_reference()[1]
        c = Chunk(aff.copy(), voxel_size=(4, 4, 4))
        Chunk(mask, voxel_size=(8, 16, 8)).maskout(c)
        return c.array

    def ref_crop(margin):
        r = H.import_reference()[1](aff.copy(), voxel_offset=(3, 2, 1)).crop_margin(margin)
        return np.concatenate([np.asarray(r.array, np.float32).ravel(), np.asarray(r.voxel_offset, np.float32)])

    rng = np.random.default_rng(seed)
    z, y, x = 5, 33, 47
    img = (rng.random((z, y, x)) ** (1 + seed) * rng.integers(60, 256)).astype(np.uint8)
    img[seed % z] //= 8
    lo, hi = [(0.01, 0.01), (0.1, 0.0), (0.0, 0.2)][seed]
    np.testing.assert_array_equal(OP.normalize_contrast(img, lo, hi, 1 + seed, 255 - 10 * seed, True),
                                  _ref(recorded, f"{seed}/normalize", ref_normalize))
    aff = rng.random((3, 4, 12, 10), dtype=np.float32)
    for mode in ("xy", "z"):
        np.testing.assert_array_equal(OP.quantize(aff, mode), _ref(recorded, f"{seed}/quantize_{mode}", lambda: ref_quantize(mode)))
    mask = rng.integers(0, 2, size=(2, 3, 5), dtype=np.uint8)
    np.testing.assert_array_equal(OP.maskout(mask, (8, 16, 8), aff, (4, 4, 4)), _ref(recorded, f"{seed}/maskout", ref_maskout))
    for k, margin in enumerate(((1, 2, 3), (0, 1, 2, 1, 0, 3))):
        a, o = OP.crop_margin(aff, (3, 2, 1), margin)
        got = np.concatenate([np.asarray(a, np.float32).ravel(), np.asarray(o, np.float32)])   # cropped values, then the offset
        np.testing.assert_array_equal(got, _ref(recorded, f"{seed}/crop_{k}", lambda: ref_crop(margin)))


def test_normalize_contrast_property_against_real_reference(recorded):
    """Randomised shapes, clip fractions and output ranges (40 seeded draws): oracle == real reference, bit for bit,
    including degenerate histograms (empty, single value, value 255 present / absent)."""
    draw = np.random.default_rng(2024)
    for k in range(40):
        z, y, x = int(draw.integers(1, 5)), int(draw.integers(1, 25)), int(draw.integers(1, 25))
        seed = int(draw.integers(0, 2 ** 31 - 1))
        lo = float(draw.choice([0.0, 0.01, 0.1, 0.5, 0.9, 1.0]))
        hi = float(draw.choice([0.0, 0.01, 0.1, 0.5, 1.0]))
        mn, mx = int(draw.integers(0, 41)), int(draw.integers(41, 256))
        kind = ["uniform", "dark", "top", "const", "zero"][k % 5]
        rng = np.random.default_rng(seed)
        if kind == "uniform":
            img = rng.integers(0, 256, (z, y, x), dtype=np.uint8)
        elif kind == "dark":
            img = rng.integers(0, 12, (z, y, x), dtype=np.uint8)
        elif kind == "top":
            img = rng.integers(250, 256, (z, y, x), dtype=np.uint8)
        elif kind == "const":
            img = np.full((z, y, x), rng.integers(0, 256), np.uint8)
        else:
            img = np.zeros((z, y, x), np.uint8)

        def ref():
            from chunkflow.chunk.image.base import Image
            im = Image(img.copy())
            with redirect_stdout(io.StringIO()), redirect_stderr(io.StringIO()):
                im.normalize_contrast(lo, hi, mn, mx, True)
            return im.array
        np.testing.assert_array_equal(OP.normalize_contrast(img, lo, hi, mn, mx, True), _ref(recorded, f"property/{k}", ref),
                                      err_msg=str((z, y, x, seed, lo, hi, mn, mx, kind)))
