"""Pins the oracle to the REAL reference classes.  Ports of the reference's own hot-path tests,
tests/flow/divid_conquer/test_inferencer.py.

What the reference computed is stored in tests/golden/reference_outputs.npz (whole arrays when small, a fixed
seeded sample of positions otherwise), so the comparison runs without the reference tree.  Where the reference
tree exists, `CFB_RECORD_REFERENCE=1 pytest tests/test_oracle_vs_reference.py` runs the real reference again and
rewrites that file."""
import io
import json
import os
import zlib
from contextlib import redirect_stdout

import numpy as np
import pytest

from oracle import inferencer_oracle as O
from oracle import reference_harness as H

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs.npz")
GOLD_FULL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_network.npz")
FULL = {"network", "network_tta"}   # network-path outputs: compared in full, bit for bit (kept in GOLD_FULL)
RECORD = os.environ.get("CFB_RECORD_REFERENCE") == "1"
SAMPLE = 512    # values kept of an array larger than this


class Store:
    """Recorded reference values by key: `agree(key, ours, theirs)` compares `ours` with the reference value, which
    `theirs()` computes when recording and the stored copy provides otherwise."""

    def __init__(self):
        self.rec = {}
        self.data = {}
        if not RECORD:
            for path in (GOLD, GOLD_FULL):
                with np.load(path) as z:
                    self.data.update({k: z[k] for k in z.files})

    def _idx(self, key, n):
        if n <= SAMPLE or key in FULL:
            return None
        rng = np.random.default_rng(zlib.crc32(key.encode()))
        return np.sort(rng.choice(n, SAMPLE, replace=False))

    def agree(self, key, ours, theirs, atol=0.0):
        if not isinstance(ours, np.ndarray):   # tuples, lists, numbers: JSON
            if RECORD:
                want = json.loads(json.dumps(theirs()))
                self.rec[key + "/j"] = np.array(json.dumps(want))
            else:
                want = json.loads(str(self.data[key + "/j"]))
            assert json.loads(json.dumps(ours)) == want, (key, ours, want)
            return
        ours = np.asarray(ours)
        if RECORD:
            t = np.asarray(theirs())
            idx = self._idx(key, t.size)
            self.rec[key + "/s"] = np.array(t.shape, np.int64)
            self.rec[key + "/v"] = t.ravel() if idx is None else t.ravel()[idx]
            if idx is not None:
                self.rec[key + "/i"] = idx
        shape = tuple(int(v) for v in (self.rec if RECORD else self.data)[key + "/s"])
        want = (self.rec if RECORD else self.data)[key + "/v"]
        assert ours.shape == shape, (key, ours.shape, shape)
        idx = self._idx(key, ours.size)
        got = ours.ravel() if idx is None else ours.ravel()[idx]
        assert got.dtype == want.dtype, (key, got.dtype, want.dtype)
        if atol:
            np.testing.assert_allclose(got, want, rtol=0, atol=atol, err_msg=key)
        else:
            assert np.array_equal(got, want), key


@pytest.fixture(scope="module")
def store():
    if RECORD and not H.available():
        pytest.fail("CFB_RECORD_REFERENCE=1 needs the reference tree (CHUNKFLOW_REFERENCE_ROOT)")
    st = Store()
    yield st
    if RECORD:
        full = {k: v for k, v in st.rec.items() if k.split("/")[0] in FULL}
        np.savez_compressed(GOLD, **{k: v for k, v in st.rec.items() if k not in full})
        np.savez_compressed(GOLD_FULL, **full)


@pytest.fixture(scope="module")
def ref():
    """(Inferencer, Chunk, PatchMask) of the real reference while recording, else None (never called)."""
    if not RECORD:
        return None
    import torch
    torch.cuda.is_available = lambda: False
    return H.import_reference()


def _run_ref(ref, chunk, offset=(0, 0, 0), **kw):
    Inferencer, Chunk, _ = ref
    with redirect_stdout(io.StringIO()):
        with Inferencer(kw.pop("model", None), None, kw.pop("input_patch_size"), **kw) as inf:
            out = inf(Chunk(chunk, voxel_offset=offset))
    return out


def _agree_chunk(store, key, o, off, theirs):
    """oracle array `o` (and voxel offset `off`) against the reference chunk `theirs()`"""
    r = {}
    def get():
        if "c" not in r:
            r["c"] = theirs()
        return r["c"]
    store.agree(key + ".offset", [int(v) for v in off], lambda: [int(v) for v in get().voxel_offset])
    store.agree(key, o, lambda: np.asarray(get().array))


def test_non_aligned_input_chunk(ref, store):  # reference test_inferencer.py:141-169 (smaller in z)
    rng = np.random.default_rng(1)
    img = rng.integers(1, 255, size=(28 + 4 + 6, 192 + 64 + 7, 192 * 2 + 64 + 9), dtype=np.uint8)
    o, off = O.infer_chunk(img, input_patch_size=(32, 256, 256), output_patch_overlap=(4, 64, 64), num_output_channels=2,
                           framework="identity")
    _agree_chunk(store, "non_aligned", o, off, lambda: _run_ref(
        ref, img, input_patch_size=(32, 256, 256), output_patch_overlap=(4, 64, 64), num_output_channels=2, batch_size=5,
        framework="identity", mask_output_chunk=True))
    np.testing.assert_allclose(img.astype(np.float32) / 255, o[0], rtol=1e-5, atol=1e-5)


def test_aligned_input_size_and_offset(ref, store):  # reference test_inferencer.py:34-58
    from chunkflow_b200 import Chunk
    image = Chunk.create(size=(18, 224, 224), dtype="uint8")   # == the reference's (test_chunk_create_sin_and_zero_...)
    o, off = O.infer_chunk(image.array, (5, 6, 7), input_patch_size=(10, 128, 128), output_patch_overlap=(2, 32, 32),
                           num_output_channels=3, framework="identity", mask_output_chunk=False)
    assert off == (7, 38, 39)
    _agree_chunk(store, "aligned_offset", o, off, lambda: _run_ref(
        ref, image.array, offset=(5, 6, 7), input_patch_size=(10, 128, 128), num_output_channels=3, output_patch_overlap=(2, 32, 32),
        input_size=(18, 224, 224), mask_output_chunk=False, framework="identity", dtype="float32"))


def test_test_time_augmentation(ref, store):  # reference test_inferencer.py:6-32
    from chunkflow_b200 import Chunk
    image = Chunk.create(size=(18, 224, 224), dtype="uint8")
    o, _ = O.infer_chunk(image.array, input_patch_size=(10, 128, 128), output_patch_overlap=(2, 32, 32),
                         num_output_channels=3, framework="identity", mask_output_chunk=False, augment=True)
    store.agree("tta_identity", o, lambda: np.asarray(_run_ref(
        ref, image.array, input_patch_size=(10, 128, 128), num_output_channels=3, output_patch_overlap=(2, 32, 32),
        input_size=(18, 224, 224), mask_output_chunk=False, framework="identity", augment=True, dtype="float32").array), atol=1e-7)


def test_network_path_bit_exact(ref, store, unet_model):
    from conftest import MODEL_FILE
    rng = np.random.default_rng(2)
    img = rng.integers(0, 256, size=(10, 36, 44), dtype=np.uint8)
    o, _ = O.infer_chunk(img, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3,
                         framework="pytorch", model=unet_model)
    store.agree("network", o, lambda: np.asarray(_run_ref(
        ref, img, model=MODEL_FILE, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3,
        batch_size=1, framework="pytorch", mask_output_chunk=True).array))


def test_myelin_and_patch_mask(ref, store):
    for ps, ov in [((10, 128, 128), (2, 32, 32)), ((8, 32, 32), (2, 8, 8))]:
        store.agree(f"patch_mask_{ps}_{ov}", O.make_patch_mask(ps, ov), lambda: np.asarray(ref[2](ps, ov)))


def test_cropped_output_patch_and_crop_margin(ref, store):
    """SURVEY section 8 f2: output patch smaller than the input patch, explicit crop margin through `patch_num`, a global
    voxel offset, no chunk-wise mask.  (The reference's own test of this configuration is skipped upstream as 'known bug',
    test_inferencer.py:98-139; with mask_output_chunk=True the reference itself produces NaN / asserts.)  The GPU path is
    compared with the oracle on exactly this configuration in tests/test_gpu_parity.py."""
    rng = np.random.default_rng(13)
    img = rng.integers(1, 256, size=(2 * 6 + 4, 2 * 24 + 16, 2 * 24 + 16), dtype=np.uint8)
    kw = dict(input_patch_size=(10, 40, 40), output_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8))
    o, off = O.infer_chunk(img, (123, 345, 567), num_output_channels=1, framework="identity", mask_output_chunk=False, **kw)
    _agree_chunk(store, "cropped", o, off, lambda: _run_ref(
        ref, img, offset=(123, 345, 567), num_output_channels=1, framework="identity", batch_size=5, mask_output_chunk=False,
        patch_num=(2, 2, 2), **kw))


def test_network_test_time_augmentation_literal(ref, store, unet_model):
    """--augment with a REAL network through the reference: its flips act on the channel / batch axes (transform.py:30-52);
    the oracle's literal mode (what the device path is tested against) reproduces the reference bit for bit."""
    from conftest import MODEL_FILE
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, size=(10, 36, 36), dtype=np.uint8)
    kw = dict(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3)
    o, _ = O.infer_chunk(img, framework="pytorch", model=unet_model, augment=True, **kw)
    store.agree("network_tta", o, lambda: np.asarray(_run_ref(
        ref, img, model=MODEL_FILE, batch_size=1, framework="pytorch", mask_output_chunk=True, augment=True, **kw).array), atol=1e-7)
    # ... and equals 1/4 (n(x) + rev_c n(x) + T n(T x) + rev_c T n(T x)): symmetric under channel reversal
    np.testing.assert_allclose(o[0], o[2], rtol=0, atol=1e-6)   # up to the order of the 8-term fp32 sum


def test_patch_mask_random_geometries_reference_native_oracle(ref, store):
    """PatchMask of the REAL reference (patch/patch_mask.py:6-68) == the native library's host code (`cfb_make_patch_mask`)
    == the oracle, bit for bit, on 60 random patch sizes / overlaps (rows a3 / a4)."""
    from chunkflow_b200 import _native
    rng = np.random.default_rng(2026)
    for k in range(60):
        ps = tuple(int(v) for v in rng.integers(2, 40, 3))
        ov = tuple(int(rng.integers(0, p // 2 + 1)) for p in ps)
        mine = O.make_patch_mask(ps, ov)
        store.agree(f"patch_mask_random_{k}", mine, lambda: np.asarray(ref[2](ps, ov)))
        assert np.array_equal(_native.make_patch_mask(ps, ov), mine), (ps, ov)


def test_identity_random_geometries_oracle_equals_reference(ref, store):
    """Whole-operator arithmetic (patch grid with clamped last patches, blend order, chunk mask, normalise) on random small
    chunk / patch / overlap combinations, identity backend: oracle == real reference, bit for bit (rows a1, a2, a5-a7, a11-a13)."""
    rng = np.random.default_rng(7)
    for k in range(12):
        ps = tuple(int(v) for v in rng.integers(4, 13, 3))
        ov = tuple(int(rng.integers(1, p // 2 + 1)) for p in ps)
        size = tuple(int(p + rng.integers(0, 2 * p)) for p in ps)
        img = rng.integers(1, 255, size=size, dtype=np.uint8)
        off = tuple(int(v) for v in rng.integers(-5, 6, 3))
        kw = dict(input_patch_size=ps, output_patch_overlap=ov, num_output_channels=int(rng.integers(1, 4)))
        bs = int(rng.integers(1, 4))
        o, o_off = O.infer_chunk(img, voxel_offset=off, framework="identity", **kw)
        _agree_chunk(store, f"identity_random_{k}", o, o_off, lambda: _run_ref(
            ref, img, offset=off, batch_size=bs, framework="identity", mask_output_chunk=True, **kw))


def test_cropped_output_random_aligned_geometries(ref, store):
    """Row f2 on random configurations: output patch smaller than the input patch (crop margin per patch), aligned chunk
    built from `patch_num`, no chunk-wise mask, random voxel offset: oracle == real reference, bit for bit."""
    rng = np.random.default_rng(31)
    for k in range(8):
        crop = tuple(int(v) for v in rng.integers(0, 4, 3))
        out_ps = tuple(int(v) for v in rng.integers(4, 11, 3))
        in_ps = tuple(o + 2 * c for o, c in zip(out_ps, crop))
        ov = tuple(int(rng.integers(1, o // 2 + 1)) for o in out_ps)
        num = tuple(int(v) for v in rng.integers(1, 4, 3))
        in_ov = tuple(2 * c + o for c, o in zip(crop, ov))
        size = tuple((p - io) * n + io for p, io, n in zip(in_ps, in_ov, num))       # reference inferencer.py:131-135
        img = rng.integers(1, 256, size=size, dtype=np.uint8)
        off = tuple(int(v) for v in rng.integers(-50, 50, 3))
        kw = dict(input_patch_size=in_ps, output_patch_size=out_ps, output_patch_overlap=ov)
        c = int(rng.integers(1, 3))
        bs = int(rng.integers(1, 4))
        o, o_off = O.infer_chunk(img, off, num_output_channels=c, framework="identity", mask_output_chunk=False, **kw)
        _agree_chunk(store, f"cropped_random_{k}", o, o_off, lambda: _run_ref(
            ref, img, offset=off, num_output_channels=c, framework="identity", batch_size=bs, mask_output_chunk=False,
            patch_num=num, **kw))


def test_myelin_threshold_and_float_input_random(ref, store):
    """`--mask-myelin-threshold` (inferencer.py:468-477 -> Chunk.mask_using_last_channel, chunk/base.py:685-689) and a float32
    input chunk (no /255), identity backend with 4 output channels, random geometry: oracle == real reference, bit for bit."""
    rng = np.random.default_rng(41)
    for k in range(6):
        ps = tuple(int(v) for v in rng.integers(4, 11, 3))
        ov = tuple(int(rng.integers(1, p // 2 + 1)) for p in ps)
        size = tuple(int(p + rng.integers(0, 2 * p)) for p in ps)
        if k % 2:
            img = rng.random(size, dtype=np.float32)
        else:
            img = rng.integers(1, 255, size=size, dtype=np.uint8)
        thr = float(rng.uniform(0.2, 0.8))
        kw = dict(input_patch_size=ps, output_patch_overlap=ov, num_output_channels=4, mask_myelin_threshold=thr)
        o, _ = O.infer_chunk(img, framework="identity", **kw)
        assert o.shape == (3,) + size
        store.agree(f"myelin_random_{k}", o, lambda: np.asarray(_run_ref(
            ref, img, framework="identity", mask_output_chunk=True, batch_size=2, **kw).array))


def test_chunk_create_sin_and_zero_match_the_reference(ref, store):
    """`create-chunk` inputs (chunk/base.py:139-199): pattern 'sin' / 'zero', uint8 and float32, 3-D and 4-D sizes: the product's
    Chunk.create == the real reference's, bit for bit (row a17; 'random' deviates by design: the reference relabels with cc3d)."""
    from chunkflow_b200 import Chunk as OurChunk
    rng = np.random.default_rng(5)
    for k in range(10):
        size = tuple(int(v) for v in rng.integers(1, 40, 3))
        if k % 3 == 2:
            size = (int(rng.integers(1, 4)),) + size
        for dtype in ("uint8", "float32"):
            for pattern in ("sin", "zero"):
                off = tuple(int(v) for v in rng.integers(-9, 9, 3))

                def want():
                    with redirect_stdout(io.StringIO()):
                        return ref[1].create(size=size, dtype=np.dtype(dtype), pattern=pattern, voxel_offset=off, voxel_size=(4, 4, 40))
                got = OurChunk.create(size=size, dtype=np.dtype(dtype), pattern=pattern, voxel_offset=off, voxel_size=(4, 4, 40))
                key = f"create_{k}_{dtype}_{pattern}"
                store.agree(key, got.array, lambda: np.asarray(want().array))
                store.agree(key + ".geometry", [list(map(int, got.voxel_offset)), list(map(int, got.voxel_size))],
                            lambda: [list(map(int, w.voxel_offset)), list(map(int, w.voxel_size))] if (w := want()) else None)


def test_chunk_glue_cutout_blend_crop_match_the_reference(ref, store):
    """Row a16: the product's host `Chunk` (cutout in global slices, blend with clipping at the buffer border, crop_margin,
    mask_using_last_channel) against the real reference's `Chunk` on random boxes (chunk/base.py:685-726,761-807)."""
    from chunkflow_b200 import Chunk as OurChunk
    RefChunk = ref[1] if ref else None
    rng = np.random.default_rng(17)
    for k in range(25):
        c = int(rng.integers(1, 4))
        size = tuple(int(v) for v in rng.integers(6, 20, 3))
        off = tuple(int(v) for v in rng.integers(-20, 20, 3))
        base = rng.random((c,) + size, dtype=np.float32)
        ours = OurChunk(base.copy(), voxel_offset=off)
        theirs = RefChunk(base.copy(), voxel_offset=off) if ref else None
        # cutout of a random inner box, global coordinates
        lo = tuple(int(rng.integers(0, s - 2)) for s in size)
        hi = tuple(int(rng.integers(l + 1, s + 1)) for l, s in zip(lo, size))
        sl = tuple(slice(o + l, o + h) for o, l, h in zip(off, lo, hi))
        a = ours.cutout(sl)
        _agree_chunk(store, f"glue_{k}_cutout", a.array, a.voxel_offset, lambda: theirs.cutout(sl))
        # blend a patch that sticks out of the buffer on some sides
        psz = tuple(int(v) for v in rng.integers(3, 10, 3))
        poff = tuple(int(o + rng.integers(-p + 1, s)) for o, p, s in zip(off, psz, size))
        patch = rng.random((c,) + psz, dtype=np.float32)
        ours.blend(OurChunk(patch.copy(), voxel_offset=poff))
        if ref:
            theirs.blend(RefChunk(patch.copy(), voxel_offset=poff))
        store.agree(f"glue_{k}_blend", ours.array, lambda: np.asarray(theirs.array))
        # crop_margin, mask_using_last_channel
        m = tuple(int(rng.integers(0, (s - 1) // 2)) for s in size)
        a = ours.crop_margin(m)
        _agree_chunk(store, f"glue_{k}_crop", a.array, a.voxel_offset, lambda: theirs.crop_margin(m))
        if c > 1:
            thr = float(rng.uniform(0.2, 0.8))
            a = OurChunk(base.copy(), voxel_offset=off).mask_using_last_channel(thr)
            _agree_chunk(store, f"glue_{k}_mask", a.array, a.voxel_offset,
                         lambda: RefChunk(base.copy(), voxel_offset=off).mask_using_last_channel(threshold=thr))


def test_transform_sequences_literal_mode_matches_the_reference(ref, store):
    """Row a15, host plug-in path: the product's TransformSequences('reference') == the real reference's
    (flow/divid_conquer/transform.py:114-156) on random 5-D buffers -- every one of the 8 forward copies and 8 backward results."""
    from chunkflow_b200.flow.divid_conquer.transform import TransformSequences
    theirs = None
    if ref:
        from chunkflow.flow.divid_conquer.transform import TransformSequences as RefTS
        theirs = RefTS()
    ours = TransformSequences('reference')
    rng = np.random.default_rng(3)
    for k in range(6):
        b, c, z, n = (int(v) for v in (rng.integers(1, 4), rng.integers(1, 4), rng.integers(1, 5), rng.integers(2, 9)))
        x = rng.random((b, c, z, n, n), dtype=np.float32)
        fo = ours.forward(x)
        ft = theirs.forward(x) if ref else [None] * 8
        assert len(fo) == 8
        for i, (p, q) in enumerate(zip(fo, ft)):
            store.agree(f"transform_{k}_forward_{i}", np.asarray(p), lambda: np.asarray(q))
        outs = [rng.random(p.shape, dtype=np.float32) for p in fo]
        bo = ours.backward([o.copy() for o in outs])
        bt = theirs.backward([o.copy() for o in outs]) if ref else [None] * len(bo)
        for i, (p, q) in enumerate(zip(bo, bt)):
            store.agree(f"transform_{k}_backward_{i}", np.asarray(p), lambda: np.asarray(q))


def test_plugin_surface_matches_the_reference(ref, store):
    """Rows a8 / a10 / B3: the plugin base class carries the attributes the reference's Inferencer reads, with the same values,
    and `Universal` drives an identity plugin of the reference's example contract (examples/inference/universal_identity.py)
    to the same per-patch result as the reference's Universal running that example."""
    import tempfile
    from chunkflow_b200.flow.divid_conquer.patch.universal import Universal
    RefUniversal = None
    if ref:
        from chunkflow.flow.divid_conquer.patch.universal import Universal as RefUniversal
    rng = np.random.default_rng(23)
    with tempfile.TemporaryDirectory() as tmp:
        plugin = os.path.join(tmp, "universal_identity.py")
        with open(plugin, "w") as f:
            f.write(EXAMPLE_PLUGIN)
        for k in range(5):
            out_ps = tuple(int(v) for v in rng.integers(4, 12, 3))
            crop = tuple(int(v) for v in rng.integers(0, 3, 3))
            in_ps = tuple(o + 2 * c for o, c in zip(out_ps, crop))
            ov = tuple(int(rng.integers(1, o // 2 + 1)) for o in out_ps)
            kw = dict(input_patch_size=in_ps, output_patch_size=out_ps, output_patch_overlap=ov, num_output_channels=1)
            ours = Universal(plugin, None, **kw)
            theirs = RefUniversal(os.path.join(H.REFERENCE_ROOT, "examples", "inference", "universal_identity.py"), None, **kw) if ref else None
            for name in ("input_patch_size", "output_patch_size", "output_patch_overlap", "num_output_channels", "crop_margin",
                         "input_patch_overlap", "input_patch_stride", "output_patch_stride"):
                store.agree(f"plugin_{k}_{name}", [int(v) for v in np.atleast_1d(getattr(ours, name))],
                            lambda: [int(v) for v in np.atleast_1d(getattr(theirs, name))])
            store.agree(f"plugin_{k}_mask", np.asarray(ours.output_patch_mask_numpy), lambda: np.asarray(theirs.output_patch_mask_numpy))
            # the example plugin multiplies by the OUTPUT patch mask: feed it a patch of the output size, like its own test does
            patch = rng.random((2, 1) + out_ps, dtype=np.float32)
            store.agree(f"plugin_{k}_call", np.asarray(ours(patch.copy())), lambda: np.asarray(theirs(patch.copy())))
            big = rng.random((1, 3) + in_ps, dtype=np.float32)
            store.agree(f"plugin_{k}_crop", np.asarray(ours._crop_output_patch(big)), lambda: np.asarray(theirs._crop_output_patch(big)))


# identity network; the plugin applies the output patch mask (the contract of the reference's example plugin)
EXAMPLE_PLUGIN = """import numpy as np


class PatchInferencer:
    def __init__(self, model_weight_file, output_patch_mask):
        self.output_patch_mask = output_patch_mask

    @property
    def compute_device(self):
        return 'cpu'

    def __call__(self, input_patch):
        output_patch = input_patch * self.output_patch_mask
        return output_patch
"""


def _reference_cli_options():
    """Options of the reference's commands (flow/flow.py:1850-1893 for `inference`), read as text: importing that module
    needs cloud packages."""
    import ast
    import re
    src = open(os.path.join(H.REFERENCE_ROOT, "chunkflow", "flow", "flow.py")).read()

    def reference_options(command):
        seg = src[src.index(f"@main.command('{command}')"):]
        seg = seg[:seg.index("\ndef ")]
        opts = []
        for m in re.finditer(r"@click\.option\((.*?)\)\s*(?=@click\.option|@operator|@generator|@main|$)", seg, re.S):
            body = m.group(1)
            flags = re.findall(r"'(-{1,2}[A-Za-z][\w/-]*)'", body.split("help=")[0])
            default = re.search(r"default=(\([^)]*\)|[^,\s)]+)", body)
            try:
                value = ast.literal_eval(default.group(1)) if default else None
            except (ValueError, SyntaxError):
                value = None     # (an expression such as Cartesian(...): only compared for `inference`, whose defaults are literals)
            opts.append([flags, list(value) if isinstance(value, tuple) else value, "required=True" in body])
        return opts
    return {c: reference_options(c) for c in ("inference", "create-chunk", "connected-components", "normalize-contrast",
                                              "crop-margin", "quantize")}


def test_cli_inference_options_match_the_reference_source(store):
    """Boundary B1: every option of the reference's `inference` command exists here with the same flags, the same default and
    the same `required` -- plus the extra `b200` framework choice.  Also `create-chunk`'s and `connected-components`' flag names."""
    from chunkflow_b200.flow import cli

    def ours(command):
        table = {}
        for p in command.params:
            for o in p.opts + p.secondary_opts:
                table[o] = p
        return table

    if RECORD:
        opts = _reference_cli_options()
        store.rec["cli_options/j"] = np.array(json.dumps(opts))
    else:
        opts = json.loads(str(store.data["cli_options/j"]))
    mine = ours(cli.inference)
    ref_opts = opts["inference"]
    assert len(ref_opts) == 19
    for flags, default, required in ref_opts:
        for f in flags:
            for part in f.split("/"):
                assert part in mine, part
        p = mine[flags[0].split("/")[0]]
        got = p.default
        if isinstance(default, list):
            got = list(got)
        assert got == default or (default is None and got in (None, ())), (flags, default, p.default)
        assert bool(p.required) == required, flags
    assert set(mine["--framework"].type.choices) == {"universal", "identity", "pytorch", "b200"}
    for command, obj in (("create-chunk", cli.create_chunk), ("connected-components", cli.connected_components),
                         ("normalize-contrast", cli.normalize_contrast), ("crop-margin", cli.crop_margin), ("quantize", cli.quantize)):
        have = ours(obj)
        for flags, _, _ in opts[command]:
            for f in flags:
                if f == "--crop-bbox/--no-crop-bbox":   # crop-margin's bounding-box bookkeeping belongs to the storage operators
                    continue
                for part in f.split("/"):
                    assert part in have, (command, part)


def test_inferencer_constructor_signature_matches_the_reference(ref, store):
    """Boundary B2: the constructor keywords of the reference's Inferencer (inferencer.py:36-54), in order, with the same
    defaults; the product appends `device` and `precision`."""
    import inspect
    from chunkflow_b200 import Inferencer as Ours

    def sig(cls):
        return [[n, None if p.default is inspect.Parameter.empty else repr(p.default), p.default is inspect.Parameter.empty]
                for n, p in inspect.signature(cls.__init__).parameters.items()]
    mine = sig(Ours)
    if RECORD:
        theirs = sig(ref[0])
        store.rec["inferencer_signature/j"] = np.array(json.dumps(theirs))
        for name in ("compute_device", "__enter__", "__exit__", "__call__"):
            assert hasattr(ref[0], name)
    else:
        theirs = json.loads(str(store.data["inferencer_signature/j"]))
    assert mine[:len(theirs)] == theirs
    assert [n for n, _, _ in mine[len(theirs):]] == ["device", "precision"]
    for name in ("compute_device", "__enter__", "__exit__", "__call__"):
        assert hasattr(Ours, name)

