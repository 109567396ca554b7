"""The plain U-Net family of convnet/unet3l.py on the CPU: the depth-3 member unchanged, the depth read back from checkpoints,
the refusals, the algorithmic FLOP counts, and the 2- and 4-level goldens of the reference's `-f pytorch` path against the
torch-CPU oracle."""
import numpy as np
import pytest

from conftest import MODEL_FILE
from oracle import inferencer_oracle as O


@pytest.fixture(scope="module")
def U():
    from chunkflow_b200.lib import load_source
    return load_source(MODEL_FILE)


def _digest(state):
    import hashlib
    h = hashlib.sha256()
    for k in sorted(state):
        h.update(k.encode())
        h.update(np.ascontiguousarray(state[k].detach().cpu().numpy().astype(np.float32)).tobytes())
    return h.hexdigest()


def test_depth3_seeded_state_is_unchanged(U, geometry):
    import torch
    if torch.__version__ != geometry["torch"]:
        pytest.skip("different torch build")
    assert _digest(U.create_model().state_dict()) == geometry["unet3l_state_sha256"]
    assert _digest(U.create_model(depth=3).state_dict()) == geometry["unet3l_state_sha256"]
    assert _digest(U.load_model(None).state_dict()) == geometry["unet3l_state_sha256"]
    assert geometry["unet3l_state_sha256"] == "50a53a77a45d9bc903585e6bb728b749109f0e2c3c179bc36ea721f13222f146"


def test_depth3_module_order_and_layer_spec(U):
    m = U.UNet3L(1, 3)
    assert list(dict(m.named_children())) == ["enc0", "enc1", "enc2", "up1", "dec1", "up0", "dec0", "head", "pool"]
    assert U.LAYER_SPEC == U.layer_spec(3)
    assert U.WIDTHS == (16, 32, 64)
    d4 = U.UNet(1, 3, depth=4)
    assert list(dict(d4.named_children())) == ["enc0", "enc1", "enc2", "enc3", "up2", "dec2", "up1", "dec1", "up0", "dec0",
                                               "head", "pool"]


@pytest.mark.parametrize("depth", [2, 3, 4])
def test_layer_spec_matches_the_state_dict(U, depth):
    state = U.create_model(depth=depth).state_dict()
    spec = U.layer_spec(depth)
    assert {f"{n}.{t}" for n, _, _, _ in spec for t in ("weight", "bias")} == set(state)
    for name, kind, cin, cout in spec:
        w = state[name + ".weight"].shape
        if kind == "convT":
            assert w == (cin, cout, 1, 2, 2)
        elif kind == "conv3":
            assert w == (cout, cin, 3, 3, 3)
        else:
            assert w == (3, cin, 1, 1, 1)


@pytest.mark.parametrize("depth", [2, 3, 4])
def test_depth_read_back_from_checkpoint(U, tmp_path, depth):
    import torch
    model = U.create_model(cout=2, seed=1, depth=depth)
    path = tmp_path / f"d{depth}.pt"
    torch.save({"state_dict": model.state_dict()}, path)
    loaded = U.load_model(str(path))
    assert loaded.depth == depth and isinstance(loaded, U.UNet)
    assert _digest(loaded.state_dict()) == _digest(model.state_dict())
    x = torch.rand(1, 1, 4, 16, 16)
    with torch.no_grad():
        assert torch.equal(loaded(x), model(x))


def _save(tmp_path, state, name):
    import torch
    path = tmp_path / name
    torch.save(state, path)
    return str(path)


def test_refusals(U, tmp_path):
    import torch
    for depth in (1, 5):
        with pytest.raises(ValueError, match="depth"):
            U.UNet(1, 3, depth=depth)
    d4 = U.create_model(depth=4).state_dict()
    d1 = {k: v for k, v in d4.items() if k.startswith(("enc0.", "head."))}
    with pytest.raises(ValueError, match="depth must be one of"):
        U.load_model(_save(tmp_path, d1, "d1.pt"))
    d5 = dict(d4)
    d5["enc4.0.weight"], d5["enc4.0.bias"] = torch.zeros(256, 128, 3, 3, 3), torch.zeros(256)
    with pytest.raises(ValueError, match="depth must be one of"):
        U.load_model(_save(tmp_path, d5, "d5.pt"))
    w48 = dict(U.create_model(depth=3).state_dict())
    w48["enc2.0.weight"] = torch.zeros(48, 32, 3, 3, 3)
    with pytest.raises(ValueError, match="widths must double from 16"):
        U.load_model(_save(tmp_path, w48, "w48.pt"))


def test_flop_counts(U):
    assert [U.flops_per_voxel(d) for d in (2, 3, 4)] == [78016, 141248, 204480]
    assert U.flops_per_voxel(3, cout=1) == 141248 - 2 * 16 * 2


def test_family_is_canonical():
    from chunkflow_b200.flow.divid_conquer.patch import b200 as b200_patch
    assert b200_patch.is_canonical_model(MODEL_FILE)


@pytest.mark.parametrize("depth", [2, 4])
def test_oracle_matches_reference_golden(U, golden, depth):
    import torch
    g = golden("unet_depth_small.npz")
    model = U.create_model(cout=3, seed=5, depth=depth)
    if torch.__version__ == str(g["torch"]):
        assert _digest(model.state_dict()) == str(g[f"state_sha256_{depth}"])
    out, _ = O.infer_chunk(g[f"input{depth}"], input_patch_size=(8, 32, 32), output_patch_overlap=(2, 8, 8),
                           num_output_channels=3, framework="pytorch", model=model)
    atol = 1e-6 if torch.__version__ == str(g["torch"]) else 1e-4
    np.testing.assert_allclose(out, g[f"output{depth}"], rtol=0, atol=atol)
    assert out.min() > 0 and out.max() < 1 and out.std() > 0.05
