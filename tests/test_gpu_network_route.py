"""The kernels each network route issues, in order, and the launch count the engine reports for them.

`bench.py` names its per-layer figures after these profiling names and reports the launch count as `gpu_launches`, so both
are pinned here for every route: the whole-chunk path in each precision route and cross-check switch, and the per-patch
plug-in path (`cfb_patch_forward_host`)."""
import math

import numpy as np
import pytest

from conftest import MODEL_FILE

pytestmark = pytest.mark.gpu

SWITCHES = ("CFB_NO_POOL_FUSION", "CFB_NO_FUSED_TAIL", "CFB_SIMT_CONVT")
PATCH, OVERLAP, BATCH = (8, 32, 32), (2, 8, 8), 3

TC = ["enc0.0", "enc0.2", "enc1.0", "enc1.2", "enc2.0", "enc2.2", "up1", "dec1.0", "dec1.2", "up0", "dec0.0"]
TC_UNFUSED_POOL = ["enc0.0", "enc0.2", "pool0", "enc1.0", "enc1.2", "pool1", "enc2.0", "enc2.2", "up1", "dec1.0", "dec1.2",
                   "up0", "dec0.0"]
SIMT = TC_UNFUSED_POOL + ["dec0.2", "head"]

CHUNK_ROUTES = {
    "tensor-core": (None, {}, TC + ["dec0.2+head+blend"]),
    "no-pool-fusion": (None, {"CFB_NO_POOL_FUSION": "1"}, TC_UNFUSED_POOL + ["dec0.2+head+blend"]),
    "no-fused-tail": (None, {"CFB_NO_FUSED_TAIL": "1"}, TC + ["dec0.2", "head+blend"]),
    "simt-convT": (None, {"CFB_SIMT_CONVT": "1"}, TC + ["dec0.2+head+blend"]),
    "f16x3": ("f16x3", {}, TC + ["dec0.2+head+blend"]),
    "simt": ("simt", {}, ["extract"] + SIMT + ["blend"]),
}
PLUGIN_ROUTES = {
    "tensor-core": (None, TC + ["dec0.2", "head"]),
    "simt": ("simt", SIMT),
}


def _inferencer(monkeypatch, precision, env):
    from chunkflow_b200 import Inferencer
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return Inferencer(MODEL_FILE, None, PATCH, output_patch_overlap=OVERLAP, num_output_channels=3, framework="b200",
                      batch_size=BATCH, mask_output_chunk=True, precision=precision)


@pytest.mark.parametrize("route", sorted(CHUNK_ROUTES))
def test_chunk_route_layers_and_launches(monkeypatch, route):
    import torch
    precision, env, per_batch = CHUNK_ROUTES[route]
    eng = _inferencer(monkeypatch, precision, env).engine
    img = np.random.default_rng(3).integers(1, 256, size=(12, 40, 48), dtype=np.uint8)
    batches = math.ceil(len(eng.patch_grid(img.shape)) / BATCH)
    assert batches > 1 and len(eng.patch_grid(img.shape)) % BATCH   # several batches, the last one partial
    d_in = torch.from_numpy(img).cuda()
    d_out = torch.empty(eng.output_shape(img.shape), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    eng.set_profiling(True)
    # all-zero test + the network per batch + normalise, and the weight volume on the first call for a chunk shape
    for weight_volume in (1, 0):
        eng.infer_chunk_device(d_in.data_ptr(), np.uint8, img.shape, d_out.data_ptr(), stream)
        torch.cuda.synchronize()
        assert eng.last_timing()["launches"] == 1 + batches * len(per_batch) + 1 + weight_volume, route
        if weight_volume:
            layers = eng.layer_timing()
            assert list(layers) == per_batch, route
            assert {name: n for name, (_, n) in layers.items()} == {name: batches for name in per_batch}, route
    eng.set_profiling(False)


@pytest.mark.parametrize("route", sorted(PLUGIN_ROUTES))
def test_plugin_route_layers(monkeypatch, route):
    precision, names = PLUGIN_ROUTES[route]
    eng = _inferencer(monkeypatch, precision, {}).engine
    patches = np.random.default_rng(4).random((BATCH, 1) + PATCH).astype(np.float32)
    eng.set_profiling(True)
    eng.patch_forward_host(patches)
    assert list(eng.layer_timing()) == names, route
    eng.set_profiling(False)
