"""Every U-Net layer kernel on its own (cfb_debug_layer_host) against torch on the CPU in float64.

The whole-network tests are weak detectors of layer bugs: the sigmoid shrinks a pre-sigmoid error at least fourfold, the
bump mask down-weights the patch border where the padding and halo code runs, and a deep error is spread over the decoder.
Here each kernel class runs alone, in every precision mode, at batch 1 and 3 (each patch with its own offset and scale, so
that a read across patches shows), on ragged extents, with the tilings forced.

Bound: the error is measured relative to the size of the summed terms, S = conv(|x|, |w|) + |b| in float64, so that it does
not depend on the input scale:  max |got - ref| / S <= EPS[mode].  The stored-output rounding of the fp16 formats is part
of it.  The f16f8 and f16 convolutions are also held to a sharper reference, their operands quantised in numpy exactly as
the code does (act_format.cuh).

f16f8 activation range (act_format.cuh): full accuracy up to |a| = 448, down to |a| ~ 2^-7.5 (measured); below, the error
grows towards fp16 level as the e4m3 corrections become subnormal (up to 2^-12.9 S at |a| <= 1.75 * 2^-12), and there the
device also departs from the operand model, which holds at |a| ~ 2^-4 and above; 448 < |a| <= 2047 keeps fp16-level
corrections; beyond 2047 an activation (and a stored output) is clamped to +-2047.  NaN stays NaN in every format and
through every pool.
"""
import math

import numpy as np
import pytest

from chunkflow_b200 import _native

pytestmark = pytest.mark.gpu

MODES = {"simt": _native.PRECISION_F32_SIMT, "f16x3": _native.PRECISION_F16X3_UMMA, "f16f8": _native.PRECISION_F16F8_UMMA,
         "f16": _native.PRECISION_F16_UMMA}
TC_MODES = ("f16x3", "f16f8", "f16")
# max |err| / S per mode, about 2x above the largest value measured over every kernel class and case of this file on one
# NVIDIA H100 80GB HBM3 (700 W power limit): simt 3.5e-7, f16x3 1.07e-6, f16f8 1.71e-5, f16 5.2e-4; each bound is below
# the next-coarser mode's measured maximum
EPS = {"simt": 2.0 ** -20, "f16x3": 2.0 ** -19, "f16f8": 2.0 ** -14.5, "f16": 2.0 ** -10}
COARSER = {"simt": "f16x3", "f16x3": "f16f8", "f16f8": "f16"}
SWITCHES = ("CFB_FORCE_ZBLOCK", "CFB_FORCE_WEIGHT_RING", "CFB_NO_POOL_FUSION", "CFB_SIMT_CONVT", "CFB_NO_FUSED_TAIL")
TILINGS = {"auto": {}, "zblock": {"CFB_FORCE_ZBLOCK": "2"}, "ring": {"CFB_FORCE_WEIGHT_RING": "1"}}

_engines = {}


def engine(mode):
    if mode not in _engines:
        _engines[mode] = _native.Engine(input_patch_size=(8, 32, 32), output_patch_size=(8, 32, 32),
                                        output_patch_overlap=(2, 8, 8), output_crop_margin=(0, 0, 0),
                                        framework=_native.FRAMEWORK_IDENTITY, precision=MODES[mode])
    return _engines[mode]


@pytest.fixture
def switches(monkeypatch):
    """Sets the kernel switches of one case (and clears the others)."""
    def set_(env):
        for k in SWITCHES:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
    return set_


# ---- inputs ------------------------------------------------------------------------------------------------------------
def activations(rng, nb, c, size, scale=1.0):
    """(nb, c, *size) float32: patch i has its own offset and scale, so that a read of the wrong patch shows."""
    x = rng.standard_normal((nb, c) + tuple(size))
    for i in range(nb):
        x[i] = x[i] * (1.0, 0.5, 2.0)[i % 3] + (0.0, 0.75, -0.5)[i % 3]
    return (x * scale).astype(np.float32)


def weights(rng, shape, fan_in):
    return (rng.standard_normal(shape) / np.sqrt(fan_in)).astype(np.float32)


# ---- float64 references --------------------------------------------------------------------------------------------
def _t(x):
    import torch
    return torch.from_numpy(np.asarray(x, np.float64))


def ref_conv3(x, w, b, relu=True):
    """(reference, S) of a 3x3x3 convolution, padding 1."""
    import torch.nn.functional as F
    y = F.conv3d(_t(x), _t(w), _t(b), padding=1)
    s = F.conv3d(_t(x).abs(), _t(w).abs(), _t(b).abs(), padding=1)
    return (y.clamp(min=0) if relu else y).numpy(), s.numpy()


def ref_convT(x, w, b):
    import torch.nn.functional as F
    y = F.conv_transpose3d(_t(x), _t(w), _t(b), stride=(1, 2, 2))
    s = F.conv_transpose3d(_t(x).abs(), _t(w).abs(), _t(b).abs(), stride=(1, 2, 2))
    return y.numpy(), s.numpy()


def pool(x):
    import torch.nn.functional as F
    return F.max_pool3d(_t(x), (1, 2, 2)).numpy()


def ref_head(x, w, b):
    """(sigmoid(head), S): the sigmoid's slope is at most 1/4, S + 1 bounds the error of the pre-sigmoid sum and the
    fp32 sigmoid itself."""
    import torch
    y = torch.einsum("bczyx,oc->bozyx", _t(x), _t(w)) + _t(b)[None, :, None, None, None]
    s = torch.einsum("bczyx,oc->bozyx", _t(x).abs(), _t(w).abs()) + _t(b).abs()[None, :, None, None, None]
    return torch.sigmoid(y).numpy(), s.numpy() + 1.0


def blend(net, out, origins, crop, mask, scale):
    """Crop every patch's output, multiply by the mask and `scale`, add into `out` at the patch's origin (clipped)."""
    out = out.astype(np.float64)
    oz, oy, ox = mask.shape
    for p, (gz, gy, gx) in zip(net, origins):
        v = p[:, crop[0]:crop[0] + oz, crop[1]:crop[1] + oy, crop[2]:crop[2] + ox] * (mask.astype(np.float64) * scale)
        z0, y0, x0 = max(gz, 0), max(gy, 0), max(gx, 0)
        z1, y1, x1 = min(gz + oz, out.shape[1]), min(gy + oy, out.shape[2]), min(gx + ox, out.shape[3])
        if z1 > z0 and y1 > y0 and x1 > x0:
            out[:, z0:z1, y0:y1, x0:x1] += v[:, z0 - gz:z1 - gz, y0 - gy:y1 - gy, x0 - gx:x1 - gx]
    return out


def ratio(got, ref, s):
    """|got - ref| / S, NaN where exactly one of them is NaN (so that max() reports it)."""
    r = np.abs(got.astype(np.float64) - ref) / np.maximum(s, 1e-300)
    same_nan = np.isnan(got) & np.isnan(ref)
    return np.where(same_nan, 0.0, np.where(np.isnan(got) | np.isnan(ref), np.inf, r))


def assert_bound(r, mode, what, eps=None):
    eps = EPS[mode] if eps is None else eps
    mx, rms = float(r.max()), float(np.sqrt(np.mean(np.square(r))))
    print(f"{what} [{mode}] max|err|/S = {mx:.3e} (2^{math.log2(mx) if mx > 0 else -math.inf:.1f})  rms = {rms:.3e}  bound {eps:.3e}")
    assert mx <= eps, f"{what} [{mode}]: max |err|/S = {mx:.3e} > {eps:.3e}"
    return mx, rms


# ---- the operand model of the f16f8 and f16 formats (act_format.cuh, pack_blocks / weight_beta in kernels_wgmma.cu) ----
def _fp16(x32):
    import torch
    return x32.to(torch.float16).to(torch.float32)


def _e4m3(x32):
    """float32 -> e4m3 -> float64.  The device converts with __NV_SATFINITE; torch's cast makes NaN of out-of-range values,
    so clamp first (NaN stays NaN)."""
    import torch
    return x32.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).to(torch.float64)


def f16f8_act(a):
    """H = fp16(clamp(32 a)), A8 = e4m3(a), L8 = e4m3(64 (32 a - H)), float64."""
    import torch
    a = torch.from_numpy(np.asarray(a, np.float32))
    s = (a * 32.0).clamp(-65504.0, 65504.0)
    h = _fp16(s)
    return h.double(), _e4m3(a), _e4m3((s - h) * 64.0)


def f16f8_wgt(w):
    """(beta, WH, WL8, W8) of one packed layer (beta = 2^14 / max|w| rounded up to a power of two)."""
    import torch
    w = torch.from_numpy(np.asarray(w, np.float32))
    wmax = float(w.abs().max())
    beta = 16384.0 / 2.0 ** math.ceil(math.log2(wmax)) if wmax > 0 and math.isfinite(wmax) else 16384.0
    wb = w * beta
    wh = _fp16(wb)
    return beta, wh.double(), _e4m3((wb - wh) * 32.0), _e4m3(w * (beta / 64.0))


def operand_model(mode, x, w, b, op="conv3", relu=True):
    """What the tensor cores compute from the quantised operands, summed in float64 (f16f8 and f16)."""
    import torch
    import torch.nn.functional as F
    conv = (lambda u, v: F.conv3d(u, v, padding=1)) if op == "conv3" else (lambda u, v: F.conv_transpose3d(u, v, stride=(1, 2, 2)))
    halves = [w] if op == "convT" or w.shape[0] <= 64 else [w[:64], w[64:]]  # cout 128: two layers of 64, each its own beta
    outs = []
    for wh_ in halves:
        if mode == "f16":
            outs.append(conv(_fp16(torch.from_numpy(x)).double(), _fp16(torch.from_numpy(wh_)).double()))
            continue
        beta, wh, wl8, w8 = f16f8_wgt(wh_)
        h, a8, l8 = f16f8_act(x)
        outs.append((conv(h, wh) + conv(a8, wl8) + conv(l8, w8)) / (32.0 * beta))
    y = torch.cat(outs, 1) + _t(b)[None, :, None, None, None]
    return (y.clamp(min=0) if relu else y).numpy()


def assert_operand_model(mode, got, model, s, what):
    """|got - model| <= rel |model| + 2^-20 S: one rounding of the stored output (f16f8 ~2^-15, fp16 one ulp) and the fp32
    accumulation order."""
    rel = 2.0 ** -14 if mode == "f16f8" else 2.0 ** -10
    excess = np.abs(got.astype(np.float64) - model) - rel * np.abs(model)
    r = np.maximum(excess, 0.0) / s
    print(f"{what} [{mode}] operand model: max (|got - model| - {rel:.1e}|model|)/S = {r.max():.3e}")
    assert r.max() <= 2.0 ** -20, what


# ---- store8 / load8 (kernels_cp8.cu) ---------------------------------------------------------------------------------
def format_round_trip(mode, v):
    """planar -> CP8 -> planar in numpy, float32 exactly as the device rounds."""
    import torch
    v32 = torch.from_numpy(np.asarray(v, np.float32))
    if mode == "f16":
        return _fp16(v32).numpy()
    if mode == "f16x3":
        hi = _fp16(v32)
        return (hi + _fp16(v32 - hi)).numpy()
    s = torch.minimum(torch.maximum(v32 * 32.0, torch.tensor(-65504.0)), torch.tensor(65504.0))  # NaN propagates
    h = _fp16(s)
    l8 = _e4m3((s - h) * 64.0).to(torch.float32)
    return ((h + l8 * (1.0 / 64.0)) * (1.0 / 32.0)).numpy()


# ---- the hook --------------------------------------------------------------------------------------------------------
def split(x, cb):
    """The concat input as two sources: the last cb channels go to the second."""
    ca = x.shape[1] - cb
    return np.ascontiguousarray(x[:, :ca]), (np.ascontiguousarray(x[:, ca:]) if cb else None)


def conv_case(mode, ca, cb, cout, size, nb=1, seed=0, scale=1.0, relu=True, model=True, x=None, eps=None):
    """One 3x3x3 convolution ca + cb -> cout; returns (max, rms) of |err| / S."""
    rng = np.random.default_rng(seed * 7919 + ca * 1000 + cb * 100 + cout + nb)
    cin = ca + cb
    x = activations(rng, nb, cin, size, scale) if x is None else x
    w = weights(rng, (cout, cin, 3, 3, 3), 27 * cin)
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    a_, b_ = split(x, cb)
    got = engine(mode).debug_layer("conv3", a_, b_, w, b, relu=relu)
    ref, s = ref_conv3(x, w, b, relu)
    what = f"conv3 {ca}+{cb}->{cout} {size} nb={nb} scale={scale}"
    res = assert_bound(ratio(got, ref, s), mode, what, eps)
    if model and mode in ("f16f8", "f16"):
        assert_operand_model(mode, got, operand_model(mode, x, w, b, relu=relu), s, what)
    return res


# (ca, cb, cout): every 3x3x3 convolution of the layer tables of depth 2, 3 and 4 (the decoders' first layers read the
# concat of two sources)
CONV_CONFIGS = [(16, 0, 16), (16, 0, 32), (32, 0, 32), (32, 0, 64), (64, 0, 64), (32, 32, 32), (16, 16, 16), (64, 0, 128),
                (128, 0, 128), (64, 64, 64)]
SIZES = [(1, 7, 9), (2, 9, 13), (5, 13, 70), (2, 8, 130), (5, 16, 40)]


def _conv_params():
    out = []
    for i, (ca, cb, cout) in enumerate(CONV_CONFIGS):
        for nb in (1, 3):
            if nb == 1 and max(ca, cb, cout) == 128:
                continue  # a 128-channel tensor is batch-major at nb = 1: always run it at nb > 1
            for mode in MODES:
                out.append(pytest.param(mode, ca, cb, cout, SIZES[(i + nb) % len(SIZES)], nb,
                                        id=f"{mode}-{ca}+{cb}-{cout}-nb{nb}"))
    return out


@pytest.mark.parametrize("mode,ca,cb,cout,size,nb", _conv_params())
def test_conv3(mode, ca, cb, cout, size, nb, switches):
    switches({})
    conv_case(mode, ca, cb, cout, size, nb)


# the extents patch >> level of the benchmark geometries 20x256x256 and 32x256x256, in the benchmarked mode
@pytest.mark.parametrize("ca,cb,cout,size,nb", [(16, 0, 16, (20, 256, 256), 1), (32, 32, 32, (32, 128, 128), 1),
                                                (64, 0, 64, (20, 64, 64), 3), (128, 0, 128, (32, 32, 32), 3),
                                                (64, 64, 64, (32, 64, 64), 2)])
def test_conv3_benchmark_extents(ca, cb, cout, size, nb, switches):
    switches({})
    conv_case("f16f8", ca, cb, cout, size, nb, model=False)


@pytest.mark.parametrize("tiling", list(TILINGS))
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("c,size,nb", [(16, (5, 14, 70), 3), (32, (2, 8, 130), 3), (64, (5, 10, 12), 3), (16, (1, 8, 8), 1),
                                       (16, (20, 128, 128), 1)])
def test_conv3_fused_pool(mode, tiling, c, size, nb, switches):
    """The 16->16, 32->32 and 64->64 layers with the (1,2,2) max pool in their epilogue (tensor cores), or a pool kernel."""
    if size[0] == 20 and (mode != "f16f8" or tiling != "auto"):
        pytest.skip("the benchmark extent runs in the benchmarked mode")
    switches(TILINGS[tiling])
    rng = np.random.default_rng(c + nb)
    x = activations(rng, nb, c, size)
    w = weights(rng, (c, c, 3, 3, 3), 27 * c)
    b = rng.standard_normal(c).astype(np.float32) * 0.1
    got, pooled = engine(mode).debug_layer("conv3_pool", x, None, w, b)
    ref, s = ref_conv3(x, w, b)
    assert_bound(ratio(got, ref, s), mode, f"conv3+pool {c} {size} nb={nb} {tiling}: activation")
    assert_bound(ratio(pooled, pool(ref), pool(s)), mode, f"conv3+pool {c} {size} nb={nb} {tiling}: pooled")


CONVT_CONFIGS = [(32, 16, (2, 9, 13), 3), (64, 32, (5, 7, 70), 3), (128, 64, (3, 8, 10), 3), (32, 16, (1, 4, 66), 1),
                 (64, 32, (16, 32, 32), 1)]


@pytest.mark.parametrize("variant", ["auto", "zblock", "ring", "simt_convT"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("ca,cout,size,nb", CONVT_CONFIGS)
def test_convT(mode, variant, ca, cout, size, nb, switches):
    """The (1,2,2) transposed convolutions: wgmma (forced tilings), CUDA cores (CFB_SIMT_CONVT), fp32 in simt mode."""
    if mode == "simt" and variant != "auto":
        pytest.skip("one fp32 kernel")
    switches({"simt_convT": {"CFB_SIMT_CONVT": "1"}}.get(variant, TILINGS.get(variant, {})))
    rng = np.random.default_rng(ca + cout + nb)
    x = activations(rng, nb, ca, size)
    w = weights(rng, (ca, cout, 1, 2, 2), ca)
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    got = engine(mode).debug_layer("convT", x, None, w, b)
    ref, s = ref_convT(x, w, b)
    what = f"convT {ca}->{cout} {size} nb={nb} {variant}"
    assert_bound(ratio(got, ref, s), mode, what)
    if mode in ("f16f8", "f16") and variant != "simt_convT":
        assert_operand_model(mode, got, operand_model(mode, x, w, b, op="convT", relu=False), s, what)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("c,size,nb", [(16, (3, 14, 70), 3), (64, (2, 8, 10), 1), (128, (2, 6, 18), 3)])
def test_maxpool(mode, c, size, nb, switches):
    switches({})
    x = activations(np.random.default_rng(c), nb, c, size)
    got = engine(mode).debug_layer("maxpool", x)
    assert_bound(ratio(got, pool(x), pool(np.abs(x))), mode, f"maxpool {c} {size} nb={nb}")


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("source,nb,size", [("patches", 1, (5, 13, 70)), ("patches", 3, (2, 9, 36)), ("uint8", 3, (4, 20, 40)),
                                            ("float32", 3, (3, 12, 36)), ("uint8", 1, (20, 256, 256))])
def test_first_layer(mode, source, nb, size, switches):
    """1 -> 16 on CUDA cores: from fp32 patches, or extracted from a uint8 (1/255) or float32 chunk at patch origins."""
    switches({})
    rng = np.random.default_rng(nb)
    w = weights(rng, (16, 1, 3, 3, 3), 27)
    b = rng.standard_normal(16).astype(np.float32) * 0.1
    if source == "patches":
        x = activations(rng, nb, 1, size)
        got = engine(mode).debug_layer("first", x, None, w, b)
    else:
        cs = (size[0] + 3, size[1] + 5, size[2] + 8)
        origins = np.array([[i % 4, (2 * i) % 6, 4 * i % 12] for i in range(nb)], np.int32)
        if source == "uint8":
            chunk = rng.integers(0, 256, cs, dtype=np.uint8)
            unit = chunk.astype(np.float32) / np.float32(255)
        else:
            chunk = rng.random(cs, dtype=np.float32)
            unit = chunk
        x = np.stack([unit[None, z:z + size[0], y:y + size[1], xx:xx + size[2]] for z, y, xx in origins])
        got = engine(mode).debug_layer("first", None, None, w, b, chunk=chunk, in_origins=origins, size=size)
    ref, s = ref_conv3(x, w, b)
    assert_bound(ratio(got, ref, s), mode, f"first {source} {size} nb={nb}")


def _head(rng, channels):
    return weights(rng, (channels, 16), 16), (rng.standard_normal(channels) * 0.5).astype(np.float32)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("channels", [1, 3, 4, 8])
@pytest.mark.parametrize("nb", [1, 3])
def test_head_sigmoid(mode, channels, nb, switches):
    switches({})
    rng = np.random.default_rng(channels * 10 + nb)
    x = np.maximum(activations(rng, nb, 16, (3, 9, 13)), 0)
    hw, hb = _head(rng, channels)
    got = engine(mode).debug_layer("head_sigmoid", x, head_weight=hw, head_bias=hb)
    ref, s = ref_head(x, hw, hb)
    assert_bound(ratio(got, ref, s), mode, f"head+sigmoid {channels} nb={nb}")


BLEND_VARIANTS = {"head_blend": ("head_blend", {}), "fused": ("conv3_head_blend", {}),
                  "fused_zblock": ("conv3_head_blend", {"CFB_FORCE_ZBLOCK": "2"}),
                  "fused_ring": ("conv3_head_blend", {"CFB_FORCE_WEIGHT_RING": "1"}),
                  "unfused_tail": ("conv3_head_blend", {"CFB_NO_FUSED_TAIL": "1"})}


def blend_case(mode, variant, channels, nb, size=(6, 20, 24), nan_at=None):
    """head + sigmoid + crop + mask + accumulate, from the 16 channels (head_blend) or after the 16 -> 16 layer."""
    op, _ = BLEND_VARIANTS[variant]
    rng = np.random.default_rng(channels * 10 + nb)
    crop = (1, 2, 3)
    out_patch = (size[0] - 2, size[1] - 4, size[2] - 6)
    x = activations(rng, nb, 16, size)
    if nan_at is not None:
        x[nan_at] = np.nan
    w = weights(rng, (16, 16, 3, 3, 3), 27 * 16)
    b = rng.standard_normal(16).astype(np.float32) * 0.1
    hw, hb = _head(rng, channels)
    mask = rng.random(out_patch, dtype=np.float32) + np.float32(0.25)
    out_size = (out_patch[0] + 3, out_patch[1] + 9, out_patch[2] + 5)
    origins = np.array([[(-1, 2, 3)[i % 3], (0, 9, -3)[i % 3], (5, 0, 2)[i % 3]] for i in range(nb)], np.int32)
    init = rng.random((channels,) + out_size, dtype=np.float32)
    scale = 0.25
    if op == "conv3_head_blend":
        act, s_act = ref_conv3(x, w, b)
        got = engine(mode).debug_layer(op, x, None, w, b, head_weight=hw, head_bias=hb, out_origins=origins,
                                       out_patch=out_patch, crop=crop, mask=mask, out=init.copy(), scale=scale)
        # the convolution's error reaches the head through |hw|: S of the head is |hw| S_act + |hb| (+ 1, ref_head)
        net, _ = ref_head(act, hw, hb)
        s_head = np.einsum("bczyx,oc->bozyx", s_act, np.abs(hw)) + np.abs(hb)[None, :, None, None, None] + 1.0
    else:
        got = engine(mode).debug_layer(op, x, head_weight=hw, head_bias=hb, out_origins=origins, out_patch=out_patch,
                                       crop=crop, mask=mask, out=init.copy(), scale=scale)
        net, s_head = ref_head(x, hw, hb)
    ref = blend(net, init, origins, crop, mask, scale)
    s = blend(s_head, np.abs(init), origins, crop, mask, scale) + np.abs(init)
    return got, ref, s


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("variant", list(BLEND_VARIANTS))
@pytest.mark.parametrize("channels,nb", [(1, 3), (3, 3), (4, 1), (8, 3), (3, 1)])
def test_head_blend(mode, variant, channels, nb, switches):
    """The head + blend on its own and fused into the epilogue of the 16 -> 16 layer (forced tilings, and unfused)."""
    if mode == "simt" and variant not in ("head_blend", "fused"):
        pytest.skip("one route in simt mode")
    switches(BLEND_VARIANTS[variant][1])
    got, ref, s = blend_case(mode, variant, channels, nb)
    assert_bound(ratio(got, ref, s), mode, f"{variant} {channels} nb={nb}")


# ---- the activation formats --------------------------------------------------------------------------------------------
def _special_values():
    rng = np.random.default_rng(1)
    v = [0.0, -0.0, 2.0 ** -24, -2.0 ** -24, 2.0 ** -20, 3 * 2.0 ** -19, 2.0 ** -15, -2.0 ** -14, 2.0 ** -9, 2.0 ** -7, 2.0 ** -6,
         448.0, -448.0, 449.0, 2047.0, -2047.0, 2048.0, 4096.0, -4096.0, 65504.0, np.nan, 1.0 / 3.0, 1e-30]
    rand = rng.choice([-1.0, 1.0], 4000) * 2.0 ** rng.uniform(-14, 11, 4000)
    return np.concatenate([np.array(v), rand, rand * 1.0000001]).astype(np.float32)


@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("c,nb", [(16, 1), (64, 3), (128, 3)])
def test_format_round_trip_bit_exact(mode, c, nb):
    """planar -> CP8 -> planar equals the numpy model of store8 / load8 bit for bit: signed zeros, fp16 and e4m3 subnormals,
    448, 2047 and beyond (f16f8: clamped to +-2047), NaN, and random values from 2^-14 to 2^11; 128 channels half-major."""
    v = _special_values()
    size = (1, 3, v.size // 3 // (c * nb) + 1)
    x = np.resize(v, (nb, c) + size).astype(np.float32)
    x.flat[:v.size] = v
    got = engine(mode).debug_layer("round_trip", x)
    want = format_round_trip(mode, x)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = np.isnan(want) | (got.view(np.uint32) == want.view(np.uint32))
    bad = np.flatnonzero(~ok)
    assert not bad.size, [(float(x.flat[i]), float(got.flat[i]), float(want.flat[i])) for i in bad[:8]]


@pytest.mark.parametrize("k", range(-12, 9))
def test_f16f8_magnitudes(k, switches):
    """The f16f8 convolution on |a| <= 1.75 * 2^k (<= 448 at k = 8): under the f16f8 bound down to k = -8, below under
    fp16's; against its operand model from k = -4 (see the module docstring)."""
    switches({})
    rng = np.random.default_rng(100 + k)
    x = (rng.uniform(-1.75, 1.75, (3, 32, 3, 9, 13)) * 2.0 ** k).astype(np.float32)
    conv_case("f16f8", 32, 0, 32, (3, 9, 13), nb=3, x=x, eps=EPS["f16f8"] if k >= -8 else EPS["f16"], model=k >= -4)


def test_f16f8_between_448_and_2047(switches):
    """448 < |a| <= 2047: A8 saturates at 448, the corrections keep fp16 level; beyond 2047 the value is clamped.  The
    weights keep the outputs below 2047, where the stored output is clamped too."""
    switches({})
    rng = np.random.default_rng(7)
    x = (rng.choice([-1.0, 1.0], (1, 16, 2, 8, 12)) * rng.uniform(448.0, 2047.0, (1, 16, 2, 8, 12))).astype(np.float32)
    w = weights(np.random.default_rng(8), (16, 16, 3, 3, 3), 27 * 16) / np.float32(8)
    b = np.zeros(16, np.float32)
    got = engine("f16f8").debug_layer("conv3", x, None, w, b, relu=False)
    ref, s = ref_conv3(x, w, b, relu=False)
    assert np.abs(ref).max() < 2047
    assert_bound(ratio(got, ref, s), "f16", "conv3 448 < |a| <= 2047 [f16f8]")
    assert_operand_model("f16f8", got, operand_model("f16f8", x, w, b, relu=False), s, "conv3 448 < |a| <= 2047")
    xc = x * 4  # 1792 <= |a| <= 8188: clamped to +-2047
    got = engine("f16f8").debug_layer("conv3", xc, None, w / np.float32(2), b, relu=False)
    ref, s = ref_conv3(np.clip(xc, -2047, 2047), w / np.float32(2), b, relu=False)
    assert np.abs(ref).max() < 2047
    assert_bound(ratio(got, ref, s), "f16", "conv3 |a| > 2047 against the clamped input [f16f8]")


# ---- the bounds separate the modes -------------------------------------------------------------------------------------
@pytest.mark.parametrize("ca,cb,cout,size,nb", [(16, 0, 16, (5, 13, 70), 3), (32, 32, 32, (2, 9, 13), 1),
                                                (64, 0, 128, (2, 8, 20), 3)])
def test_bounds_order_the_modes(ca, cb, cout, size, nb, switches):
    """On one case, rms |err|/S orders the modes (f16x3 < f16f8 / 4, f16f8 < f16 / 8): a partly dropped or wrongly scaled
    correction term fails at any input scale.  Each mode's bound fails on the next-coarser mode's output."""
    switches({})
    rng = np.random.default_rng(ca + cb + cout)
    x = activations(rng, nb, ca + cb, size)
    w = weights(rng, (cout, ca + cb, 3, 3, 3), 27 * (ca + cb))
    b = rng.standard_normal(cout).astype(np.float32) * 0.1
    ref, s = ref_conv3(x, w, b)
    a_, b_ = split(x, cb)
    r = {m: ratio(engine(m).debug_layer("conv3", a_, b_, w, b), ref, s) for m in MODES}
    rms = {m: float(np.sqrt(np.mean(np.square(v)))) for m, v in r.items()}
    print("rms |err|/S", rms, "max", {m: float(v.max()) for m, v in r.items()})
    order = [("simt", "f16x3", 2), ("f16x3", "f16f8", 4), ("f16f8", "f16", 8)]
    for fine, coarse, f in order:
        assert rms[fine] < rms[coarse] / f, (fine, coarse, rms)
        assert not rms[coarse] < rms[fine] / f  # the check run against the next-coarser mode fails
    for m in MODES:
        assert r[m].max() <= EPS[m], m
    # simt and f16x3 overlap in their maxima (fp32 accumulation against ~22-bit operands): the rms order separates them
    for m in ("f16x3", "f16f8"):
        assert r[COARSER[m]].max() > EPS[m], f"the {m} bound passes the {COARSER[m]} output"


# ---- NaN -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("path", ["fused", "unfused", "maxpool"])
def test_nan_reaches_the_pooled_output(mode, path, switches):
    """One NaN in a (1,2,2) window makes that pooled voxel NaN (torch.max_pool3d), on every pool path; a NaN input voxel
    makes every output of its 3x3x3 neighbourhood NaN."""
    switches({"CFB_NO_POOL_FUSION": "1"} if path == "unfused" else {})
    rng = np.random.default_rng(3)
    c, size, nb = 16, (3, 8, 10), 3
    x = activations(rng, nb, c, size)
    x[1, 5, 1, 3, 4] = np.nan
    if path == "maxpool":
        got = engine(mode).debug_layer("maxpool", x)
        want = pool(x)
    else:
        w = np.abs(weights(rng, (c, c, 3, 3, 3), 27 * c))
        b = np.full(c, 0.5, np.float32)
        act, got = engine(mode).debug_layer("conv3_pool", x, None, w, b)
        ref, _ = ref_conv3(x, w, b)
        assert np.array_equal(np.isnan(act), np.isnan(ref)) and np.isnan(act[1, :, 0:3, 2:5, 3:6]).all()
        want = pool(ref)
    assert np.isnan(want).any() and np.array_equal(np.isnan(got), np.isnan(want))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("variant", ["head_blend", "fused", "unfused_tail"])
def test_nan_survives_head_and_blend(mode, variant, switches):
    """A NaN activation reaches the blended output chunk, so that the output range check still fires."""
    if mode == "simt" and variant == "unfused_tail":
        pytest.skip("one route in simt mode")
    switches(BLEND_VARIANTS[variant][1])
    got, ref, _ = blend_case(mode, variant, 3, 3, nan_at=(0, 4, 2, 5, 7))
    assert np.isnan(ref).any() and np.array_equal(np.isnan(got), np.isnan(ref))
