"""Parity tests proper: the CUDA path, called through the C-ABI, against the CPU oracle,
the golden vectors of the real reference, and size-independent properties."""
import os

import numpy as np
import pytest

from conftest import MODEL_FILE
from chunkflow_b200 import Chunk, _native
from oracle import inferencer_oracle as O

pytestmark = pytest.mark.gpu

# identity / blend arithmetic is fp32 with atomics in arbitrary order: ~1 ulp of the sums
BLEND_ATOL = 2e-6
# fp32 SIMT convolutions vs torch-CPU: different summation order only
NET_ATOL_SIMT = 2e-5
# default mode 'f16f8' (wgmma: fp16 main product + one e4m3 K=32 product carrying both hi/lo correction terms, fp32
# accumulate): measured 0.9e-4 .. 2.1e-4; the bar in BASELINE.json's north_star is 1e-3 max-abs -- assert 2x tighter
NET_ATOL_F32 = 5e-4
# 'f16x3' (fp16 hi/lo split, three products per multiply): measured 2e-5 .. 5e-5 -- assert 5x tighter than the bar
NET_ATOL_X3 = 2e-4
NET_ATOL = 1e-3
# single-pass fp16 (reference --dtype float16): operands and stored activations carry 11 bits
NET_ATOL_F16 = 2e-2


def _inferencer(**kw):
    from chunkflow_b200 import Inferencer
    return Inferencer(kw.pop("model", None), kw.pop("weights", None), kw.pop("input_patch_size"), **kw)


def test_patch_grid_through_the_c_abi(geometry):
    for key, starts in geometry["patch_grids"].items():
        size, patch, ov = (tuple(map(int, t.split("x"))) for t in key.split("_"))
        eng = _native.Engine(input_patch_size=patch, output_patch_size=patch, output_patch_overlap=ov,
                             output_crop_margin=(0, 0, 0), framework=_native.FRAMEWORK_IDENTITY)
        assert eng.patch_grid(size).tolist() == starts, key
        assert np.array_equal(eng.patch_mask(), O.make_patch_mask(patch, ov))
        eng.close()


def test_identity_nonaligned_golden(golden):
    g = golden("identity_nonaligned.npz")
    inf = _inferencer(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=2,
                      batch_size=5, framework="identity", mask_output_chunk=True)
    out = inf(Chunk(g["input"], voxel_offset=(3, 5, 7)))
    assert tuple(out.voxel_offset) == tuple(g["voxel_offset"])
    np.testing.assert_allclose(out.array, g["output"], rtol=0, atol=BLEND_ATOL)
    got = [[[s.start, s.stop] for s in pair[0]] + [[s.start, s.stop] for s in pair[1]] for pair in inf.patch_slices_list]
    assert got == g["patch_slices"].tolist()
    assert "H100" in inf.compute_device or "NVIDIA" in inf.compute_device


def test_identity_aligned_golden(golden):
    g = golden("identity_aligned.npz")
    inf = _inferencer(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=2,
                      patch_num=(2, 2, 2), framework="identity", batch_size=3, mask_output_chunk=False)
    out = inf(Chunk(g["input"]))
    assert tuple(out.voxel_offset) == (2, 8, 8) and out.shape == g["output"].shape
    np.testing.assert_allclose(out.array, g["output"], rtol=0, atol=BLEND_ATOL)


def test_reference_test_non_aligned_input_chunk():
    """tests/flow/divid_conquer/test_inferencer.py:141-169 at the reference's own sizes."""
    rng = np.random.default_rng(7)
    img = rng.integers(1, 255, size=(28 * 2 + 4 + 6, 192 * 2 + 64 + 7, 192 * 2 + 64 + 9), dtype=np.uint8)
    inf = _inferencer(input_patch_size=(32, 256, 256), output_patch_overlap=(4, 64, 64), num_output_channels=2,
                      batch_size=5, framework="identity", mask_output_chunk=True)
    out = inf(Chunk(img))
    np.testing.assert_allclose(img.astype(np.float32) / 255, out.array[0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out.array[0], out.array[1], rtol=0, atol=BLEND_ATOL)
    o, _ = O.infer_chunk(img, input_patch_size=(32, 256, 256), output_patch_overlap=(4, 64, 64), num_output_channels=2,
                         framework="identity")
    np.testing.assert_allclose(out.array, o, rtol=0, atol=BLEND_ATOL)


def test_reference_test_aligned_patch_num_float16():
    """test_inferencer.py:60-95: dtype float16, batch 5, two channels, aligned, no chunk mask."""
    rng = np.random.default_rng(8)
    img = rng.integers(1, 255, size=(28 * 2 + 4, 192 * 2 + 64, 192 * 2 + 64), dtype=np.uint8)
    inf = _inferencer(input_patch_size=(32, 256, 256), output_patch_overlap=(4, 64, 64), num_output_channels=2,
                      patch_num=(2, 2, 2), framework="identity", dtype="float16", batch_size=5, mask_output_chunk=False)
    out = inf(Chunk(img))
    ref = img[4:-4, 64:-64, 64:-64].astype(np.float32) / 255
    np.testing.assert_allclose(ref, out.array[0], rtol=1e-3, atol=1e-3)


def test_reference_test_time_augmentation_identity():
    """test_inferencer.py:6-32."""
    image = Chunk.create(size=(18, 224, 224), dtype="uint8")
    inf = _inferencer(input_patch_size=(10, 128, 128), num_output_channels=3, output_patch_overlap=(2, 32, 32),
                      input_size=(18, 224, 224), mask_output_chunk=False, framework="identity", augment=True)
    out = inf(image)
    assert np.all(np.isclose(image.array[2:-2, 32:-32, 32:-32], out.array[0] * 255, atol=1))
    o, _ = O.infer_chunk(image.array, input_patch_size=(10, 128, 128), output_patch_overlap=(2, 32, 32),
                         num_output_channels=3, framework="identity", mask_output_chunk=False, augment=True)
    np.testing.assert_allclose(out.array, o, rtol=0, atol=BLEND_ATOL)


@pytest.mark.parametrize("precision,dtype,atol", [(None, "float32", NET_ATOL_F32), ("simt", "float32", NET_ATOL_SIMT),
                                                  ("f16x3", "float32", NET_ATOL_X3), ("f16f8", "float32", NET_ATOL_F32),
                                                  (None, "float16", NET_ATOL_F16)])
def test_unet3l_golden(golden, precision, dtype, atol):
    """The reference's own `-f pytorch` CPU output (golden) against every precision mode."""
    g = golden("unet3l_small.npz")
    for batch in (1, 4):
        inf = _inferencer(model=MODEL_FILE, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8),
                          num_output_channels=3, batch_size=batch, framework="pytorch", mask_output_chunk=True,
                          precision=precision, dtype=dtype)
        out = inf(Chunk(g["input"]))
        err = np.abs(out.array - g["output"]).max()
        print("unet3l golden max-abs", precision, dtype, err)
        assert err <= atol


def test_unet3l_readme_config_against_oracle(unet_model):
    """BASELINE config #1 geometry (patch 20x256x256, overlap 4x64x64) on the sin chunk, 2 z-rows."""
    chunk = Chunk.create(size=(36, 256, 256), dtype=np.uint8, pattern="sin")
    inf = _inferencer(input_patch_size=(20, 256, 256), output_patch_overlap=(4, 64, 64), num_output_channels=3,
                      batch_size=2, framework="b200", mask_output_chunk=True)
    out = inf(chunk)
    o, _ = O.infer_chunk(chunk.array, input_patch_size=(20, 256, 256), output_patch_overlap=(4, 64, 64),
                         num_output_channels=3, framework="pytorch", model=unet_model)
    err = np.abs(out.array - o).max()
    print("config #1 geometry max-abs", err, "timing", inf.timing)
    assert err <= NET_ATOL_F32
    assert inf.timing["launches"] > 0


def _conv3_case(prec, cin, cout, size, atol, round_operands=False):
    import torch
    rng = np.random.default_rng(cin * 100 + cout)
    x = rng.standard_normal((cin,) + size).astype(np.float32)
    w = (rng.standard_normal((cout, cin, 3, 3, 3)) / np.sqrt(27 * cin)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    eng = _native.Engine(input_patch_size=(8, 32, 32), output_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8),
                         output_crop_margin=(0, 0, 0), framework=_native.FRAMEWORK_IDENTITY, precision=prec)
    got = eng.debug_conv3(x, w, b, relu=True)
    xt, wt = torch.from_numpy(x), torch.from_numpy(w)
    ref = torch.relu(torch.nn.functional.conv3d(xt[None], wt, torch.from_numpy(b), padding=1))[0].numpy()
    np.testing.assert_allclose(got, ref, rtol=0, atol=atol)


@pytest.mark.parametrize("cin,cout,size", [(1, 16, (5, 20, 36)), (16, 16, (4, 16, 70)), (48, 32, (3, 9, 13)), (64, 64, (6, 8, 8))])
def test_conv3_layer_simt_against_torch(cin, cout, size):
    _conv3_case(_native.PRECISION_F32_SIMT, cin, cout, size, 2e-5)


# (cin, cout, size): dense M tiles with junk columns, row-aligned 128-voxel tiles with two x tiles,
# two-source (concat) inputs, ragged x/y extents, every channel configuration of the network
UMMA_CASES = [(16, 16, (3, 8, 40)), (16, 16, (4, 16, 70)), (32, 32, (3, 12, 20)), (16, 32, (2, 6, 128)),
              (16, 16, (5, 20, 256)), (64, 64, (6, 8, 8)), (64, 32, (4, 16, 16)), (32, 16, (3, 8, 130)), (32, 64, (3, 9, 64)),
              (16, 16, (2, 7, 9))]


@pytest.mark.parametrize("cin,cout,size", UMMA_CASES)
def test_conv3_layer_tcgen05_split_against_torch(cin, cout, size):
    # hi/lo split operands: ~22 significant bits, fp32 accumulation
    _conv3_case(_native.PRECISION_F16X3_UMMA, cin, cout, size, 5e-5)


@pytest.mark.parametrize("zstack", ["2", "3", "4", "8"])
@pytest.mark.parametrize("cin,cout,size", [(16, 16, (3, 8, 40)), (16, 16, (9, 16, 70)), (32, 32, (5, 12, 20)), (16, 32, (4, 6, 128)),
                                           (32, 16, (7, 8, 130)), (64, 32, (4, 16, 16)), (16, 16, (1, 7, 9))])
def test_conv3_layer_tcgen05_zstacked_kernel(monkeypatch, zstack, cin, cout, size):
    """The convolution split along z into blocks of T output planes per CTA (each block loads its own halo planes), forced."""
    monkeypatch.setenv("CFB_FORCE_ZBLOCK", zstack)
    _conv3_case(_native.PRECISION_F16X3_UMMA, cin, cout, size, 5e-5)
    if cin == 16:
        _conv3_case(_native.PRECISION_F16_UMMA, cin, cout, size, 1e-2)


@pytest.mark.parametrize("zstack", ["2", "3", "4"])
@pytest.mark.parametrize("cin,cout,size", [(16, 16, (3, 8, 40)), (16, 16, (9, 16, 70)), (32, 32, (5, 12, 20)), (16, 32, (4, 6, 128)),
                                           (32, 16, (7, 8, 130)), (64, 32, (4, 16, 16)), (16, 16, (1, 7, 9))])
def test_conv3_layer_tcgen05_tmem_shift_kernel(monkeypatch, zstack, cin, cout, size):
    """z blocks of T output planes with the weights streamed through a 3-stage ring (taps refilled while the MMAs run)
    instead of resident, forced."""
    monkeypatch.setenv("CFB_FORCE_ZBLOCK", zstack)
    monkeypatch.setenv("CFB_FORCE_WEIGHT_RING", "1")
    _conv3_case(_native.PRECISION_F16X3_UMMA, cin, cout, size, 5e-5)
    if cin == 16:
        _conv3_case(_native.PRECISION_F16_UMMA, cin, cout, size, 1e-2)


@pytest.mark.parametrize("cin,cout,size", UMMA_CASES)
def test_conv3_layer_tcgen05_f16f8_against_torch(cin, cout, size):
    # fp16 main product + one e4m3 (K = 32) product for both correction terms: ~2^-16 relative per product
    # (inputs ~N(0,1), outputs of magnitude ~5: fp16 alone is asserted at 1e-2 below, the hi/lo split at 5e-5)
    _conv3_case(_native.PRECISION_F16F8_UMMA, cin, cout, size, 4e-4)


@pytest.mark.parametrize("zstack", ["2", "3", "4"])
@pytest.mark.parametrize("cin,cout,size", [(16, 16, (9, 16, 70)), (32, 32, (5, 12, 20)), (64, 32, (4, 16, 16)), (16, 16, (1, 7, 9))])
def test_conv3_layer_f16f8_forced_zstack(monkeypatch, zstack, cin, cout, size):
    monkeypatch.setenv("CFB_FORCE_ZBLOCK", zstack)
    _conv3_case(_native.PRECISION_F16F8_UMMA, cin, cout, size, 4e-4)


@pytest.mark.parametrize("cin,cout,size", UMMA_CASES[:4])
def test_conv3_layer_tcgen05_fp16_against_torch(cin, cout, size):
    # single-pass fp16: 11-bit operands and 11-bit stored outputs on values of magnitude ~5
    _conv3_case(_native.PRECISION_F16_UMMA, cin, cout, size, 1e-2)


def test_plugin_level_patch_inferencer(unet_model):
    """B3: per-patch numpy API, output already cropped and masked (reference patch/pytorch.py:98-119)."""
    from chunkflow_b200.flow.divid_conquer.patch.b200 import B200
    rng = np.random.default_rng(11)
    patches = rng.random((3, 1, 8, 32, 32)).astype(np.float32)
    pi = B200(MODEL_FILE, None, (8, 32, 32), (8, 32, 32), (2, 8, 8), num_output_channels=3, batch_size=2)
    got = pi(patches)
    geom = O.Geometry((8, 32, 32), None, (2, 8, 8))
    ref = np.concatenate([O.TorchPatch(geom, 3, O.make_patch_mask((8, 32, 32), (2, 8, 8)), unet_model)(p[None]) for p in patches])
    np.testing.assert_allclose(got, ref, rtol=0, atol=NET_ATOL_F32)
    # ... and as framework='prebuilt' inside the Inferencer (device extract/blend around a host plugin)
    img = rng.integers(0, 256, size=(12, 40, 48), dtype=np.uint8)
    inf = _inferencer(model=pi, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3,
                      batch_size=2, framework="prebuilt")
    out = inf(Chunk(img))
    o, _ = O.infer_chunk(img, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3,
                         framework="pytorch", model=unet_model)
    np.testing.assert_allclose(out.array, o, rtol=0, atol=NET_ATOL_F32)


def test_universal_plugin_file(tmp_path):
    """`-f universal` with the reference's example plugin contract (examples/inference/universal_identity.py)."""
    plugin = tmp_path / "universal_identity.py"
    plugin.write_text(
        "import numpy as np\n"
        "class PatchInferencer:\n"
        "    def __init__(self, model_weight_file, output_patch_mask):\n"
        "        self.output_patch_mask = output_patch_mask\n"
        "    @property\n"
        "    def compute_device(self):\n"
        "        return 'host-plugin'\n"
        "    def __call__(self, input_patch):\n"
        "        out = np.copy(input_patch) * self.output_patch_mask\n"
        "        return np.repeat(out, 3, axis=1)\n")
    image = Chunk.create(size=(36, 448, 448), dtype="uint8")
    inf = _inferencer(model=str(plugin), input_patch_size=(20, 256, 256), output_patch_overlap=(4, 64, 64),
                      patch_num=(2, 2, 2), framework="universal", batch_size=3, mask_output_chunk=False,
                      num_output_channels=3)
    out = inf(image)
    assert inf.compute_device == "host-plugin" and out.shape == (3, 28, 320, 320)
    np.testing.assert_allclose(image.array[4:-4, 64:-64, 64:-64].astype(np.float32) / 255, out.array[2], atol=1e-5)


def test_edge_cases_zero_input_range_check_myelin_dry_run(unet_model):
    kw = dict(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), batch_size=3)
    # all-zero shortcut (reference inferencer.py:387-393): zeros even though sigmoid(net(0)) != 0
    inf = _inferencer(model=MODEL_FILE, num_output_channels=3, framework="b200", **kw)
    out = inf(Chunk(np.zeros((10, 40, 40), np.uint8)))
    assert out.shape == (3, 10, 40, 40) and not out.array.any()
    # a chunk of exactly one patch
    one = inf(Chunk.create(size=(8, 32, 32)))
    o, _ = O.infer_chunk(Chunk.create(size=(8, 32, 32)).array, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8),
                         num_output_channels=3, framework="pytorch", model=unet_model)
    np.testing.assert_allclose(one.array, o, rtol=0, atol=NET_ATOL_F32)
    # chunk smaller than a patch: refused (reference asserts iz >= 0, inferencer.py:270-271)
    with pytest.raises(_native.NativeError):
        inf(Chunk.create(size=(6, 32, 32)))
    # float input > 1 through identity trips the reference's `< 1.0001` assertion (inferencer.py:465-466)
    ident = _inferencer(num_output_channels=1, framework="identity", **kw)
    with pytest.raises(AssertionError):
        ident(Chunk(np.full((10, 40, 40), 1.5, np.float32)))
    ok = ident(Chunk(np.full((10, 40, 40), 0.25, np.float32)))
    np.testing.assert_allclose(ok.array, 0.25, atol=BLEND_ATOL)
    # myelin masking needs 4 channels, returns 3 (reference inferencer.py:468-477, chunk/base.py:685-689)
    rng = np.random.default_rng(5)
    img = rng.random((10, 40, 40)).astype(np.float32)
    my = _inferencer(num_output_channels=4, framework="identity", mask_myelin_threshold=0.5, **kw)
    res = my(Chunk(img))
    assert res.shape == (3, 10, 40, 40)
    np.testing.assert_allclose(res.array[0], np.where(img < 0.5, img, 0), atol=BLEND_ATOL)
    # dry run returns a synthetic chunk of the output shape without touching the device path
    dry = _inferencer(num_output_channels=2, framework="identity", dry_run=True, **kw)(Chunk.create(size=(10, 40, 40)))
    assert dry.shape == (2, 10, 40, 40)
    # uint16 input is normalised by its dtype maximum
    u16 = (rng.random((10, 40, 40)) * 65535).astype(np.uint16)
    r16 = ident(Chunk(u16))
    np.testing.assert_allclose(r16.array[0], u16.astype(np.float32) / 65535, atol=BLEND_ATOL)


def test_cropped_output_patch_and_crop_margin(unet_model):
    """output_patch_size < input_patch_size with an explicit output crop margin and a global offset.
    (The reference's own test for this is skipped upstream as 'known bug', test_inferencer.py:98-139;
    the oracle restates the arithmetic as written.)"""
    rng = np.random.default_rng(13)
    img = rng.integers(1, 256, size=(2 * 6 + 4, 2 * 24 + 16, 2 * 24 + 16), dtype=np.uint8)
    kw = dict(input_patch_size=(10, 40, 40), output_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8))
    inf = _inferencer(num_output_channels=1, framework="identity", batch_size=5, mask_output_chunk=False,
                      patch_num=(2, 2, 2), **kw)
    out = inf(Chunk(img, voxel_offset=(123, 345, 567)))
    o, off = O.infer_chunk(img, (123, 345, 567), num_output_channels=1, framework="identity", mask_output_chunk=False, **kw)
    assert tuple(out.voxel_offset) == off and out.shape == o.shape
    np.testing.assert_allclose(out.array, o, rtol=0, atol=BLEND_ATOL)


def test_large_chunk_properties():
    """Size-independent properties at a larger size than the oracle handles quickly: the blend of
    an identity network reproduces the input (partition of unity + normalisation), is channel-
    symmetric and idempotent across repeated calls with cached tables."""
    rng = np.random.default_rng(17)
    img = rng.integers(1, 255, size=(96, 600, 520), dtype=np.uint8)
    inf = _inferencer(input_patch_size=(32, 256, 256), output_patch_overlap=(8, 64, 64), num_output_channels=3,
                      batch_size=12, framework="identity")
    a = inf(Chunk(img)).array
    np.testing.assert_allclose(a[0], img.astype(np.float32) / 255, rtol=1e-5, atol=1e-5)
    assert np.abs(a[0] - a[2]).max() <= BLEND_ATOL
    b = inf(Chunk(img)).array
    assert np.abs(a - b).max() <= BLEND_ATOL


def test_cli_readme_example(golden):
    """README config #1 through the command line: create-chunk 64x256x256 -> inference (b200)."""
    from click.testing import CliRunner
    from chunkflow_b200.flow import cli
    res = CliRunner().invoke(cli.main, [
        "create-chunk", "--size", "40", "256", "256",
        "inference", "--input-patch-size", "20", "256", "256", "--output-patch-overlap", "4", "64", "64",
        "--num-output-channels", "3", "--framework", "b200", "--batch-size", "2", "--mask-output-chunk"],
        standalone_mode=False)
    assert res.exception is None, res.output
    task = res.return_value[0]
    out = task["chunk"]
    assert out.shape == (3, 40, 256, 256) and 0 < out.array.min() and out.array.max() < 1
    assert "inference" in task["log"]["timer"] and "H100" in task["log"]["compute_device"]


def test_slab_entry_point_matches_whole_chunk():
    """cfb_infer_slab_device + cfb_normalize_device (the per-rank half of BASELINE config #5): two z-slabs run
    one after the other on one GPU, halo planes added on the host, equal the whole-chunk result."""
    import torch
    from chunkflow_b200 import distributed as D
    rng = np.random.default_rng(23)
    img = rng.integers(1, 255, size=(27, 40, 44), dtype=np.uint8)
    inf = _inferencer(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=2,
                      batch_size=4, framework="identity")
    whole = inf(Chunk(img)).array
    eng = inf.engine
    slabs = D.plan_z_slabs(27, 8, 2, 2)
    acc = np.zeros((2, 27, 40, 44), np.float32)
    wsum = np.zeros((27, 40, 44), np.float32)
    for s in slabs:
        sub = np.ascontiguousarray(img[s.z0:s.z1])
        d_in = torch.from_numpy(sub).cuda()
        shape = eng.output_shape(sub.shape)
        part = torch.empty(shape, dtype=torch.float32, device="cuda")
        w = torch.empty(shape[1:], dtype=torch.float32, device="cuda")
        eng.infer_slab_device(d_in.data_ptr(), sub.dtype, sub.shape, 0, s.row_end - s.row_begin, part.data_ptr(), w.data_ptr())
        torch.cuda.synchronize()
        acc[:, s.z0:s.z1] += part.cpu().numpy()
        wsum[s.z0:s.z1] += w.cpu().numpy()
    d_acc, d_w = torch.from_numpy(acc).cuda(), torch.from_numpy(wsum).cuda()
    eng.normalize_device(d_acc.data_ptr(), d_w.data_ptr(), d_acc.shape)
    torch.cuda.synchronize()
    np.testing.assert_allclose(d_acc.cpu().numpy(), whole, rtol=0, atol=BLEND_ATOL)


@pytest.mark.parametrize("precision", [None, "simt"])
@pytest.mark.parametrize("augment", [True, "spatial"])
def test_device_test_time_augmentation(unet_model, precision, augment):
    """--augment on the device network path.  `augment=True` reproduces the REFERENCE's arithmetic (its FlipLR / FlipUD
    act on the channel / batch axes, transform.py:30-52: two network evaluations, each blended with its channel-reversed
    copy) and is checked against the oracle's literal mode, which tests/test_oracle_vs_reference.py pins to the real
    reference; `augment='spatial'` is the explicit opt-in with 8 spatial variants."""
    rng = np.random.default_rng(29)
    img = rng.integers(0, 256, size=(10, 40, 44), dtype=np.uint8)
    kw = dict(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3)
    inf = _inferencer(model=MODEL_FILE, framework="b200", batch_size=8, augment=augment, precision=precision, **kw)
    out = inf(Chunk(img))
    o, _ = O.infer_chunk(img, framework="pytorch", model=unet_model, augment=augment, **kw)
    plain, _ = O.infer_chunk(img, framework="pytorch", model=unet_model, **kw)
    err = np.abs(out.array - o).max()
    print("device TTA max-abs", augment, precision, err, "| TTA changes the result by", np.abs(o - plain).max())
    assert err <= (NET_ATOL_F32 if precision is None else NET_ATOL_SIMT)
    assert np.abs(o - plain).max() > 1e-2   # the augmentation is not a no-op for a real network
    if augment is True:   # the reference's average is symmetric under channel reversal
        np.testing.assert_allclose(out.array[0], out.array[2], rtol=0, atol=1e-6)


def test_host_plugin_test_time_augmentation_reference_literal(unet_model):
    """--augment around a host patch plug-in (framework='prebuilt'): transform.py in its reference-literal mode."""
    from chunkflow_b200.flow.divid_conquer.patch.b200 import B200
    rng = np.random.default_rng(37)
    img = rng.integers(0, 256, size=(10, 40, 44), dtype=np.uint8)
    kw = dict(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3)
    pi = B200(MODEL_FILE, None, (8, 32, 32), (8, 32, 32), (2, 8, 8), num_output_channels=3, batch_size=1)
    out = _inferencer(model=pi, framework="prebuilt", batch_size=1, augment=True, **kw)(Chunk(img))
    o, _ = O.infer_chunk(img, framework="pytorch", model=unet_model, augment=True, **kw)
    assert np.abs(out.array - o).max() <= NET_ATOL_F32


# ---- parity at the BENCHMARKED geometry (BASELINE configs #2 / #3: the tilings, the batch of 12 patches in flight and the
# ---- cross-patch fp32 reductions the headline number runs with) ------------------------------------------------------
def _oracle_threads():
    import torch
    try:
        import psutil
        n = psutil.cpu_count(logical=False) or 1
    except Exception:
        n = max(1, (os.cpu_count() or 2) // 2)
    n = min(n, len(os.sched_getaffinity(0)))
    torch.set_num_threads(max(1, n))


def _bench_geometry_case(unet_model, chunk_shape, patch, overlap, batch, seed):
    _oracle_threads()
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, size=chunk_shape, dtype=np.uint8)
    o, _ = O.infer_chunk(img, input_patch_size=patch, output_patch_overlap=overlap, num_output_channels=3,
                         framework="pytorch", model=unet_model)
    for precision, atol in ((None, NET_ATOL_F32), ("f16x3", NET_ATOL_X3)):   # the default (benchmarked) mode and the hi/lo split
        inf = _inferencer(model=MODEL_FILE, input_patch_size=patch, output_patch_overlap=overlap, num_output_channels=3,
                          batch_size=batch, framework="b200", mask_output_chunk=True, precision=precision)
        out = np.array(inf(Chunk(img)).array)
        err = float(np.abs(out - o).max())
        print("bench-geometry parity", chunk_shape, patch, "patches", len(inf.patch_slices_list), "batch", batch, precision, "max-abs", err)
        assert out.shape == o.shape and err <= atol
        again = inf(Chunk(img)).array    # cached tables, autotuned tilings: same result up to the order of the fp32 reductions
        assert np.abs(again - out).max() <= 1e-5


def test_bench_geometry_config3_batch12(unet_model):
    """Patch 32x256x256, overlap 8x64x64, exactly 12 patches = one full batch of the benchmark configuration (#3)."""
    _bench_geometry_case(unet_model, (80, 448, 448), (32, 256, 256), (8, 64, 64), 12, 101)


def test_bench_geometry_config3_clamped_chunk(unet_model):
    """Same patch geometry on a chunk whose last patch per axis is clamped back (heavily overlapping patches in flight)."""
    _bench_geometry_case(unet_model, (40, 300, 260), (32, 256, 256), (8, 64, 64), 12, 102)


@pytest.mark.slow
def test_bench_geometry_config2_crop_128x512x512(unet_model):
    """BASELINE config #2's geometry (patch 20x256x256, overlap 4x64x64, batch 12) on a 128x512x512 crop: 72 patches
    (SURVEY section 8d asks for full-volume parity on 'a <=128x512x512 crop-config of #2')."""
    _bench_geometry_case(unet_model, (128, 512, 512), (20, 256, 256), (4, 64, 64), 12, 103)


def test_nan_and_overflow_trip_the_range_check():
    """The reference's `assert np.all(out < 1.0001)` (inferencer.py:465-466) raises on NaN too; so must the device check."""
    ident = _inferencer(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=1, batch_size=3,
                        framework="identity")
    bad = np.full((10, 40, 40), 0.5, np.float32)
    bad[3, 7, 9] = np.nan
    with pytest.raises(AssertionError):
        ident(Chunk(bad))
    bad[3, 7, 9] = np.inf
    with pytest.raises(AssertionError):
        ident(Chunk(bad))
    bad[3, 7, 9] = 0.5
    assert np.isfinite(ident(Chunk(bad)).array).all()
    # a NaN weight makes every network output NaN
    from chunkflow_b200.flow.divid_conquer.patch import b200 as b200_patch
    inf = _inferencer(model=MODEL_FILE, input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3,
                      batch_size=2, framework="b200")
    state = dict(b200_patch.load_state_dict(MODEL_FILE, None))
    w = np.array(state["dec0.2.weight"], dtype=np.float32, copy=True)
    w.flat[5] = np.nan
    state["dec0.2.weight"] = w
    inf.engine.load_state_dict(state)
    with pytest.raises(AssertionError):
        inf(Chunk.create(size=(8, 32, 32)))


def test_host_plugin_shape_errors_and_myelin_zero_threshold():
    """ADVICE r1: a plug-in that returns a wrongly shaped array must raise (the native side would read out of bounds);
    mask_myelin_threshold=0.0 means 'off', as in the reference (truthiness, inferencer.py:468)."""
    class Uncropped:
        compute_device = "host"
        def __call__(self, patch):   # forgets to crop to the output patch
            return np.repeat(patch, 2, axis=1)
    kw = dict(input_patch_size=(10, 40, 40), output_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8))
    inf = _inferencer(model=Uncropped(), num_output_channels=2, framework="prebuilt", batch_size=2, **kw)
    with pytest.raises(ValueError):
        inf(Chunk.create(size=(16, 64, 64)))

    class TooFewChannels:
        compute_device = "host"
        def __call__(self, patch):
            return patch[:, :, 1:-1, 4:-4, 4:-4]
    inf = _inferencer(model=TooFewChannels(), num_output_channels=2, framework="prebuilt", batch_size=2, **kw)
    with pytest.raises(ValueError):
        inf(Chunk.create(size=(16, 64, 64)))
    with pytest.raises(ValueError):   # non-square patch with --augment around a host plug-in
        _inferencer(model=TooFewChannels(), input_patch_size=(8, 32, 40), output_patch_overlap=(2, 8, 8), num_output_channels=1,
                    framework="prebuilt", augment=True)
    rng = np.random.default_rng(5)
    img = rng.random((10, 40, 40)).astype(np.float32)
    my = _inferencer(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=4, framework="identity",
                     mask_myelin_threshold=0.0, batch_size=3)
    res = my(Chunk(img))
    assert res.shape == (4, 10, 40, 40)
    np.testing.assert_allclose(res.array[0], img, atol=BLEND_ATOL)


def test_kernel_variants_agree(monkeypatch, unet_model):
    """Every kernel variant computes the same network: fused vs unfused head+blend tail, first layer with its weights in the constant
    bank vs in shared memory, 3x3x3 convolutions split into z blocks, weights streamed through a ring, pooling fused into the
    convolution epilogue vs its own kernel, tensor-core vs CUDA-core transposed convolutions (forced through env switches)."""
    rng = np.random.default_rng(31)
    img = rng.integers(0, 256, size=(20, 96, 104), dtype=np.uint8)
    kw = dict(input_patch_size=(16, 64, 64), output_patch_overlap=(4, 16, 16), num_output_channels=3, framework="b200",
              batch_size=5, precision="f16x3")
    ref, _ = O.infer_chunk(img, input_patch_size=(16, 64, 64), output_patch_overlap=(4, 16, 16), num_output_channels=3,
                           framework="pytorch", model=unet_model)
    results = {}
    for name, env in [("default", {}), ("unfused_tail", {"CFB_NO_FUSED_TAIL": "1"}), ("smem_first", {"CFB_FIRST_CONV_SMEM_W": "1"}),
                      ("zblock4", {"CFB_FORCE_ZBLOCK": "4"}), ("weight_ring", {"CFB_FORCE_WEIGHT_RING": "1"}),
                      ("zblock2_ring", {"CFB_FORCE_ZBLOCK": "2", "CFB_FORCE_WEIGHT_RING": "1"}),
                      ("unfused_pool", {"CFB_NO_POOL_FUSION": "1"}), ("simt_convT", {"CFB_SIMT_CONVT": "1"})]:
        for k in ("CFB_NO_FUSED_TAIL", "CFB_FIRST_CONV_SMEM_W", "CFB_FORCE_ZBLOCK", "CFB_FORCE_WEIGHT_RING", "CFB_NO_POOL_FUSION",
                  "CFB_SIMT_CONVT"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        results[name] = _inferencer(model=MODEL_FILE, **kw)(Chunk(img)).array
        err = np.abs(results[name] - ref).max()
        print(name, "max-abs vs oracle", err)
        assert err <= NET_ATOL_X3, name
    for name, arr in results.items():
        assert np.abs(arr - results["default"]).max() <= 5e-5, name


def test_f16f8_unfused_and_cuda_core_paths(monkeypatch, unet_model):
    """The default f16f8 number format through the kernels that are not on the default route: the unfused head+blend tail, the
    first layer with shared-memory weights, the stand-alone pool and the CUDA-core transposed convolution (they decode / encode the
    H + A8 + L8 records through load8 / store8, kernels_cp8.cu)."""
    rng = np.random.default_rng(41)
    img = rng.integers(0, 256, size=(20, 96, 104), dtype=np.uint8)
    kw = dict(input_patch_size=(16, 64, 64), output_patch_overlap=(4, 16, 16), num_output_channels=3, framework="b200", batch_size=5)
    ref, _ = O.infer_chunk(img, input_patch_size=(16, 64, 64), output_patch_overlap=(4, 16, 16), num_output_channels=3,
                           framework="pytorch", model=unet_model)
    for env in ({}, {"CFB_NO_FUSED_TAIL": "1"}, {"CFB_FIRST_CONV_SMEM_W": "1"}, {"CFB_FORCE_ZBLOCK": "2"}, {"CFB_FORCE_WEIGHT_RING": "1"},
                {"CFB_NO_POOL_FUSION": "1"}, {"CFB_SIMT_CONVT": "1"}):
        for k in ("CFB_NO_FUSED_TAIL", "CFB_FIRST_CONV_SMEM_W", "CFB_FORCE_ZBLOCK", "CFB_FORCE_WEIGHT_RING", "CFB_NO_POOL_FUSION",
                  "CFB_SIMT_CONVT"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        out = _inferencer(model=MODEL_FILE, **kw)(Chunk(img)).array
        err = np.abs(out - ref).max()
        print("f16f8", env, "max-abs vs oracle", err)
        assert err <= NET_ATOL_F32, env


def test_network_on_float_and_uint16_chunks(unet_model):
    """Input chunks that are not uint8 take the CUDA-core first layer (float32 input): float32 in [0, 1] as is, wider integers
    normalised by their dtype maximum like the reference (inferencer.py:395-399)."""
    rng = np.random.default_rng(43)
    kw = dict(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3)
    inf = _inferencer(model=MODEL_FILE, framework="b200", batch_size=3, **kw)
    f = rng.random((12, 40, 48)).astype(np.float32)
    o, _ = O.infer_chunk(f, framework="pytorch", model=unet_model, **kw)
    assert np.abs(inf(Chunk(f)).array - o).max() <= NET_ATOL_F32
    u16 = (rng.random((12, 40, 48)) * 65535).astype(np.uint16)
    o16, _ = O.infer_chunk(u16, framework="pytorch", model=unet_model, **kw)
    assert np.abs(inf(Chunk(u16)).array - o16).max() <= NET_ATOL_F32
