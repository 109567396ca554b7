"""The 2- and 4-level U-Nets on the H100: the reference's `-f pytorch` goldens in every precision mode, the 20x256x256
geometry, each 128-channel layer on its own, the cross-check switches, the other entry points and the refusals."""
import numpy as np
import pytest

from conftest import MODEL_FILE
from chunkflow_b200 import Chunk, _native
from oracle import inferencer_oracle as O
from test_gpu_parity import NET_ATOL_F16, NET_ATOL_F32, NET_ATOL_SIMT, NET_ATOL_X3

pytestmark = pytest.mark.gpu

SEED = 5  # tests/golden/make_golden_unet_depth.py
KW = dict(input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8), num_output_channels=3)
SWITCHES = ("CFB_NO_POOL_FUSION", "CFB_NO_FUSED_TAIL", "CFB_SIMT_CONVT")


def _model(depth, cout=3):
    from chunkflow_b200.lib import load_source
    return load_source(MODEL_FILE).create_model(cout=cout, seed=SEED, depth=depth)


@pytest.fixture(scope="module")
def checkpoint(tmp_path_factory):
    import torch
    paths = {}
    for depth in (2, 4):
        paths[depth] = str(tmp_path_factory.mktemp("unet") / f"unet{depth}.pt")
        torch.save(_model(depth).state_dict(), paths[depth])
    return paths


def _inferencer(weights, framework="pytorch", **kw):
    from chunkflow_b200 import Inferencer
    kw = {**KW, **kw}
    return Inferencer(MODEL_FILE, weights, kw.pop("input_patch_size"), framework=framework, mask_output_chunk=True, **kw)


@pytest.mark.parametrize("depth", [2, 4])
@pytest.mark.parametrize("precision,dtype,atol", [(None, "float32", NET_ATOL_F32), ("simt", "float32", NET_ATOL_SIMT),
                                                  ("f16x3", "float32", NET_ATOL_X3), ("f16f8", "float32", NET_ATOL_F32),
                                                  (None, "float16", NET_ATOL_F16)])
def test_reference_golden(golden, checkpoint, depth, precision, dtype, atol):
    g = golden("unet_depth_small.npz")
    for batch in (1, 4):
        inf = _inferencer(checkpoint[depth], batch_size=batch, precision=precision, dtype=dtype)
        out = inf(Chunk(g[f"input{depth}"]))
        err = np.abs(out.array - g[f"output{depth}"]).max()
        print(f"depth {depth} golden max-abs", precision, dtype, batch, err)
        assert err <= atol


def test_depth4_readme_geometry_against_oracle(checkpoint):
    """Patch 20x256x256, overlap 4x64x64 (BASELINE config #1) on the sin chunk, two z rows."""
    chunk = Chunk.create(size=(36, 256, 256), dtype=np.uint8, pattern="sin")
    inf = _inferencer(checkpoint[4], framework="b200", input_patch_size=(20, 256, 256), output_patch_overlap=(4, 64, 64),
                      batch_size=2)
    out = inf(chunk)
    o, _ = O.infer_chunk(chunk.array, input_patch_size=(20, 256, 256), output_patch_overlap=(4, 64, 64),
                         num_output_channels=3, framework="pytorch", model=_model(4))
    err = np.abs(out.array - o).max()
    print("depth 4 config #1 geometry max-abs", err, "timing", inf.timing)
    assert err <= NET_ATOL_F32


@pytest.mark.parametrize("mode", ["simt", "f16x3", "f16f8", "f16"])
@pytest.mark.parametrize("cin,cout,size", [(64, 128, (3, 9, 13)), (128, 128, (4, 16, 16)), (128, 64, (3, 8, 20)),
                                           (64, 64, (5, 6, 10))])
def test_wide_layer_against_torch(mode, cin, cout, size):
    """One layer through cfb_debug_layer_host against the float64 reference and bound of test_gpu_layers.py, at three
    patches when a tensor has 128 channels (stored half-major); for cin >= 32 the input is fed as two separately allocated
    halves, so 128 -> 64 is also the decoder's 64 + 64 concat."""
    from test_gpu_layers import conv_case
    conv_case(mode, cin // 2, cin // 2, cout, size, nb=3 if 128 in (cin, cout) else 1)


def _run(monkeypatch, checkpoint, env, img, precision=None, batch=3):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k in env:
        monkeypatch.setenv(k, "1")
    inf = _inferencer(checkpoint[4], framework="b200", batch_size=batch, precision=precision)
    inf.engine.set_profiling(True)
    out = inf(Chunk(img)).array
    layers = inf.engine.layer_timing()
    inf.engine.set_profiling(False)
    return out, layers


def test_depth4_cross_check_switches(monkeypatch, checkpoint):
    """The fused 64 -> 64 pool, the wgmma and CUDA-core 128 -> 64 transposed convolutions and the fused tail agree with
    the kernels that cross-check them, and every route with the torch-CPU oracle."""
    img = np.random.default_rng(3).integers(1, 256, size=(12, 40, 48), dtype=np.uint8)
    ref, _ = O.infer_chunk(img, framework="pytorch", model=_model(4), **KW)
    base, layers = _run(monkeypatch, checkpoint, (), img)
    assert list(layers) == ["enc0.0", "enc0.2", "enc1.0", "enc1.2", "enc2.0", "enc2.2", "enc3.0", "enc3.2", "up2", "dec2.0",
                            "dec2.2", "up1", "dec1.0", "dec1.2", "up0", "dec0.0", "dec0.2+head+blend"]
    assert np.abs(base - ref).max() <= NET_ATOL_F32
    for env, names in ((("CFB_NO_POOL_FUSION",), {"pool0", "pool1", "pool2"}), (("CFB_SIMT_CONVT",), set()),
                       (("CFB_NO_FUSED_TAIL",), {"dec0.2", "head+blend"}), (SWITCHES, {"pool2", "head+blend"})):
        out, layers = _run(monkeypatch, checkpoint, env, img)
        assert names <= set(layers), (env, list(layers))
        err, dev = np.abs(out - ref).max(), np.abs(out - base).max()
        print("depth 4", env, "max-abs against the oracle", err, "against the production route", dev)
        assert err <= NET_ATOL_F32 and dev <= NET_ATOL_F32, env
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


def test_depth4_infer_device_and_augment(checkpoint):
    from chunkflow_b200.chunk.device import DeviceChunk
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, size=(10, 40, 44), dtype=np.uint8)
    inf = _inferencer(checkpoint[4], framework="b200")
    host = inf(Chunk(img, voxel_offset=(1, 2, 3)))
    dev = inf.infer_device(DeviceChunk.from_chunk(Chunk(img, voxel_offset=(1, 2, 3))))
    assert tuple(dev.voxel_offset) == tuple(host.voxel_offset)
    np.testing.assert_allclose(dev.to_chunk().array, host.array, rtol=0, atol=2e-6)
    aug = _inferencer(checkpoint[4], framework="b200", batch_size=8, augment=True)(Chunk(img)).array
    o, _ = O.infer_chunk(img, framework="pytorch", model=_model(4), augment=True, **KW)
    err = np.abs(aug - o).max()
    print("depth 4 --augment max-abs", err)
    assert err <= NET_ATOL_F32


def test_depth4_cli(checkpoint):
    from click.testing import CliRunner
    from chunkflow_b200.flow import cli
    res = CliRunner().invoke(cli.main, [
        "create-chunk", "--size", "36", "256", "256",
        "inference", "--input-patch-size", "20", "256", "256", "--output-patch-overlap", "4", "64", "64",
        "--num-output-channels", "3", "--framework", "pytorch", "-m", MODEL_FILE, "-w", checkpoint[4],
        "--batch-size", "2", "--mask-output-chunk"], standalone_mode=False)
    assert res.exception is None, res.output
    out = res.return_value[0]["chunk"]
    assert out.shape == (3, 36, 256, 256) and 0 < out.array.min() and out.array.max() < 1


def _engine(patch=(8, 32, 32)):
    return _native.Engine(input_patch_size=patch, output_patch_size=patch, output_patch_overlap=(2, 8, 8),
                          output_crop_margin=(0, 0, 0), num_output_channels=3, framework=_native.FRAMEWORK_UNET3L)


def _state(depth):
    return {k: v.numpy() for k, v in _model(depth).state_dict().items()}


def test_refusals():
    d4 = _state(4)
    cases = [({k: v for k, v in d4.items() if k.startswith(("enc0.", "head."))}, "depth must be 2, 3 or 4"),
             ({**d4, "enc4.0.weight": np.zeros((256, 128, 3, 3, 3), np.float32), "enc4.0.bias": np.zeros(256, np.float32)},
              "depth must be 2, 3 or 4"),
             ({**_state(3), "enc2.0.weight": np.zeros((48, 32, 3, 3, 3), np.float32)}, "widths must be 16, 32, 64, 128")]
    for state, msg in cases:
        eng = _engine()
        with pytest.raises(_native.NativeError, match=msg):
            eng.load_state_dict(state)
        eng.close()
    eng = _engine((8, 36, 36))
    with pytest.raises(_native.NativeError, match="patch y and x must be multiples of 8"):
        eng.load_state_dict(d4)
    eng.close()
    eng = _engine((8, 36, 36))
    eng.load_state_dict(_state(3))  # 36 is a multiple of 4: the 3-level network runs on this patch
    eng.close()
