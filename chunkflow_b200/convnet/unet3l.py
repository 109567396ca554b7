"""The plain 3D U-Net family for the ``inference`` hot path (SURVEY.md section 7.2).

The reference ships no network definition: ``-f pytorch`` loads a user file that must
expose ``load_model(weight_path)`` or ``InstantiatedModel`` (plus optional
``pre_process`` / ``post_process``), see reference
``chunkflow/flow/divid_conquer/patch/pytorch.py:48-83``.  This file satisfies that
contract, so the SAME file drives

* the reference's own ``-f pytorch`` CPU path (the parity oracle), and
* the device path, which reads the ``state_dict`` (its depth from the ``enc{k}.0`` names)
  and packs the weights into the device layout of the hand-written sm_90a kernels.

It must stay self-contained (no package-relative imports): the reference executes it
through ``SourceFileLoader("Model", fname)`` (``chunkflow/lib/__init__.py:5-16``).

Architecture: depth d in {2, 3, 4}, widths (16, 32, ..., 16 * 2**(d-1)), pooling (1, 2, 2).
Depth 3 (:class:`UNet3L`, the default) is

    enc0: conv3x3x3(1->16)+ReLU, conv3x3x3(16->16)+ReLU          full resolution
    pool (1,2,2)
    enc1: conv3x3x3(16->32)+ReLU, conv3x3x3(32->32)+ReLU         1/2 in y,x
    pool (1,2,2)
    enc2: conv3x3x3(32->64)+ReLU, conv3x3x3(64->64)+ReLU         1/4 in y,x
    up1 : convT(64->32, kernel=stride=(1,2,2)); concat [up1, enc1] -> 64
    dec1: conv3x3x3(64->32)+ReLU, conv3x3x3(32->32)+ReLU
    up0 : convT(32->16, kernel=stride=(1,2,2)); concat [up0, enc0] -> 32
    dec0: conv3x3x3(32->16)+ReLU, conv3x3x3(16->16)+ReLU
    head: conv1x1x1(16->cout) + sigmoid

Depth 2 stops after enc1; depth 4 adds enc3 (64->128, 128->128, 1/8 in y,x), up2 (128->64)
and dec2 (128->64, 64->64).  Patch y and x must be multiples of 2**(d-1).
All 3x3x3 convolutions use zero padding 1 (SAME) at the *patch* border.
FLOP per patch voxel for cout=3 (:func:`flops_per_voxel`): 78 016 (depth 2), 141 248 (depth 3),
204 480 (depth 4).  This is not RSUNet: no residual blocks, no normalisation.
"""
import math

import torch
import torch.nn as nn

DEPTHS = (2, 3, 4)
POOL = (1, 2, 2)


def widths(depth: int = 3) -> tuple:
    """Channels of the levels: 16, 32, ... doubling with every (1,2,2) pool."""
    return tuple(16 << k for k in range(depth))


WIDTHS = widths(3)


def layer_spec(depth: int = 3) -> tuple:
    """(name, kind, cin, cout) in execution order; the device path generates the same table from the state dict."""
    w = widths(depth)
    spec = []
    for k in range(depth):
        spec += [(f"enc{k}.0", "conv3", w[k - 1] if k else 1, w[k]), (f"enc{k}.2", "conv3", w[k], w[k])]
    for k in range(depth - 2, -1, -1):
        spec += [(f"up{k}", "convT", w[k + 1], w[k]),
                 (f"dec{k}.0", "conv3", 2 * w[k], w[k]), (f"dec{k}.2", "conv3", w[k], w[k])]
    spec.append(("head", "conv1", w[0], None))
    return tuple(spec)


# the default (3-level) network's layers
LAYER_SPEC = layer_spec(3)


def flops_per_voxel(depth: int = 3, cout: int = 3) -> int:
    """Algorithmic FLOP (2 per multiply-add) per input patch voxel; the max pools are not counted."""
    total = 0
    for name, kind, ci, co in layer_spec(depth):
        if kind == "conv1":
            total += 2 * ci * cout
            continue
        level = int(name[3]) if name.startswith(("enc", "dec")) else int(name[2:])
        taps = 27 if kind == "conv3" else 1  # a transposed convolution: one tap per output voxel (at its output level)
        total += 2 * taps * ci * co * 4 ** (depth - 1 - level) // 4 ** (depth - 1)
    return total


def _block(cin, cout):
    return nn.Sequential(
        nn.Conv3d(cin, cout, 3, padding=1), nn.ReLU(inplace=True),
        nn.Conv3d(cout, cout, 3, padding=1), nn.ReLU(inplace=True),
    )


class UNet(nn.Module):
    """Modules are registered enc0 .. enc{d-1}, up{d-2}, dec{d-2} .. up0, dec0, head, pool: the seeded
    initialisation draws in this order."""

    def __init__(self, cin: int = 1, cout: int = 3, depth: int = 3):
        super().__init__()
        if depth not in DEPTHS:
            raise ValueError(f"U-Net depth must be one of {DEPTHS}, got {depth}")
        self.depth = depth
        w = widths(depth)
        for k in range(depth):
            setattr(self, f"enc{k}", _block(w[k - 1] if k else cin, w[k]))
        for k in range(depth - 2, -1, -1):
            setattr(self, f"up{k}", nn.ConvTranspose3d(w[k + 1], w[k], kernel_size=POOL, stride=POOL))
            setattr(self, f"dec{k}", _block(2 * w[k], w[k]))
        self.head = nn.Conv3d(w[0], cout, 1)
        self.pool = nn.MaxPool3d(POOL)

    def forward(self, x):
        enc = []
        for k in range(self.depth):
            x = getattr(self, f"enc{k}")(self.pool(x) if k else x)
            enc.append(x)
        for k in range(self.depth - 2, -1, -1):
            x = getattr(self, f"dec{k}")(torch.cat([getattr(self, f"up{k}")(x), enc[k]], dim=1))
        # sigmoid is required: the reference asserts output < 1.0001
        # (chunkflow/flow/divid_conquer/inferencer.py:465-466)
        return torch.sigmoid(self.head(x))


class UNet3L(UNet):
    """The 3-level member, widths (16, 32, 64)."""

    def __init__(self, cin: int = 1, cout: int = 3):
        super().__init__(cin, cout, depth=3)


def seeded_init(model: nn.Module, seed: int = 0, head_gain: float = 4.0) -> nn.Module:
    """Deterministic variance-preserving init so that outputs span (0, 1).

    PyTorch's default init yields outputs in ~[0.45, 0.55], a weak parity
    discriminator (SURVEY.md 7.3).  Kaiming-normal (gain sqrt 2) on the ReLU convs,
    unit-gain on the transposed convs, a wider head, small random biases.
    """
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, m in model.named_modules():
            if isinstance(m, nn.ConvTranspose3d):
                fan_in = m.weight.shape[0]  # one tap per output voxel
                m.weight.normal_(0.0, math.sqrt(1.0 / fan_in), generator=g)
                m.bias.uniform_(-0.05, 0.05, generator=g)
            elif isinstance(m, nn.Conv3d):
                fan_in = m.weight[0].numel()
                gain = head_gain if name == "head" else math.sqrt(2.0)
                m.weight.normal_(0.0, gain / math.sqrt(fan_in), generator=g)
                m.bias.uniform_(-0.05, 0.05, generator=g)
    return model


def create_model(cin: int = 1, cout: int = 3, seed: int = 0, depth: int = 3) -> nn.Module:
    return seeded_init(UNet(cin, cout, depth), seed=seed).eval()


def state_depth(state) -> int:
    """The depth of a state dict (its ``enc{k}.0.weight`` tensors), checked against the family: 2 to 4 levels,
    level k ``16 << k`` channels wide."""
    depth = 0
    while f"enc{depth}.0.weight" in state:
        depth += 1
    if depth not in DEPTHS:
        raise ValueError(f"U-Net depth must be one of {DEPTHS}: the checkpoint has {depth} encoder levels")
    for k, w in enumerate(widths(depth)):
        got = tuple(state[f"enc{k}.0.weight"].shape)[0]
        if got != w:
            raise ValueError(f"U-Net widths must double from 16 ({widths(depth)}): enc{k}.0 has {got} channels")
    return depth


def load_model(weight_path=None, cin: int = 1, cout: int = 3):
    """Entry point used by the reference ``-f pytorch`` loader (pytorch.py:50-51).

    ``weight_path`` None/"" -> the seeded random 3-level init (there are no trained weights
    offline); otherwise a ``state_dict`` or ``{'state_dict': ...}`` checkpoint of any depth of the family.
    """
    if not weight_path:
        return create_model(cin, cout)
    chkpt = torch.load(weight_path, map_location="cpu")
    state = chkpt["state_dict"] if "state_dict" in chkpt else chkpt
    depth = state_depth(state)
    cout = state["head.weight"].shape[0]
    cin = state["enc0.0.weight"].shape[1]
    model = UNet(cin, cout, depth)
    model.load_state_dict(state)
    return model.eval()
