"""Canonical 3-level 3D U-Net for the ``inference`` hot path (SURVEY.md section 7.2).

The reference ships no network definition: ``-f pytorch`` loads a user file that must
expose ``load_model(weight_path)`` or ``InstantiatedModel`` (plus optional
``pre_process`` / ``post_process``), see reference
``chunkflow/flow/divid_conquer/patch/pytorch.py:48-83``.  This file satisfies that
contract, so the SAME file drives

* the reference's own ``-f pytorch`` CPU path (the parity oracle), and
* the device path, which reads :data:`LAYER_SPEC` / the ``state_dict`` and packs the
  weights into the device layout of the hand-written sm_90a kernels.

It must stay self-contained (no package-relative imports): the reference executes it
through ``SourceFileLoader("Model", fname)`` (``chunkflow/lib/__init__.py:5-16``).

Architecture (fixed): widths (16, 32, 64), pooling (1, 2, 2)

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

All 3x3x3 convolutions use zero padding 1 (SAME) at the *patch* border.
141 248 FLOP per patch voxel for cout=3.
"""
import math

import torch
import torch.nn as nn

WIDTHS = (16, 32, 64)
POOL = (1, 2, 2)

# (name, kind, cin, cout) in execution order; the device path packs weights by name.
LAYER_SPEC = (
    ("enc0.0", "conv3", 1, 16), ("enc0.2", "conv3", 16, 16),
    ("enc1.0", "conv3", 16, 32), ("enc1.2", "conv3", 32, 32),
    ("enc2.0", "conv3", 32, 64), ("enc2.2", "conv3", 64, 64),
    ("up1", "convT", 64, 32),
    ("dec1.0", "conv3", 64, 32), ("dec1.2", "conv3", 32, 32),
    ("up0", "convT", 32, 16),
    ("dec0.0", "conv3", 32, 16), ("dec0.2", "conv3", 16, 16),
    ("head", "conv1", 16, None),
)


def _block(cin, cout):
    return nn.Sequential(
        nn.Conv3d(cin, cout, 3, padding=1), nn.ReLU(inplace=True),
        nn.Conv3d(cout, cout, 3, padding=1), nn.ReLU(inplace=True),
    )


class UNet3L(nn.Module):
    def __init__(self, cin: int = 1, cout: int = 3):
        super().__init__()
        w0, w1, w2 = WIDTHS
        self.enc0 = _block(cin, w0)
        self.enc1 = _block(w0, w1)
        self.enc2 = _block(w1, w2)
        self.up1 = nn.ConvTranspose3d(w2, w1, kernel_size=POOL, stride=POOL)
        self.dec1 = _block(2 * w1, w1)
        self.up0 = nn.ConvTranspose3d(w1, w0, kernel_size=POOL, stride=POOL)
        self.dec0 = _block(2 * w0, w0)
        self.head = nn.Conv3d(w0, cout, 1)
        self.pool = nn.MaxPool3d(POOL)

    def forward(self, x):
        e0 = self.enc0(x)
        e1 = self.enc1(self.pool(e0))
        e2 = self.enc2(self.pool(e1))
        d1 = self.dec1(torch.cat([self.up1(e2), e1], dim=1))
        d0 = self.dec0(torch.cat([self.up0(d1), e0], dim=1))
        # sigmoid is required: the reference asserts output < 1.0001
        # (chunkflow/flow/divid_conquer/inferencer.py:465-466)
        return torch.sigmoid(self.head(d0))


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


def create_model(cin: int = 1, cout: int = 3, seed: int = 0) -> nn.Module:
    return seeded_init(UNet3L(cin, cout), seed=seed).eval()


def load_model(weight_path=None, cin: int = 1, cout: int = 3):
    """Entry point used by the reference ``-f pytorch`` loader (pytorch.py:50-51).

    ``weight_path`` None/"" -> the seeded random init (there are no trained weights
    offline); otherwise a ``state_dict`` or ``{'state_dict': ...}`` checkpoint.
    """
    if not weight_path:
        return create_model(cin, cout)
    chkpt = torch.load(weight_path, map_location="cpu")
    state = chkpt["state_dict"] if "state_dict" in chkpt else chkpt
    cout = state["head.weight"].shape[0]
    cin = state["enc0.0.weight"].shape[1]
    model = UNet3L(cin, cout)
    model.load_state_dict(state)
    return model.eval()
