"""Patch backends that run on the GPU through the C-ABI.

``B200``     : the U-Net forward (depth 2 to 4, from the weights) + crop + bump mask on the device, with the
               per-patch numpy API of the reference's ``PyTorch`` backend
               (chunkflow/flow/divid_conquer/patch/pytorch.py:10-119).  Usable as
               ``Inferencer(framework='prebuilt', convnet_model=B200(...))`` -- also inside
               the reference's own Inferencer.
``Identity`` : reference patch/identity.py:6-51 on the device (test backend).

Whole-chunk inference does not go through this per-patch API (8 MB in + 25 MB out over
PCIe per patch); ``Inferencer`` keeps the chunk resident on the device instead.
"""
from __future__ import annotations

import os

import numpy as np

from chunkflow_b200 import _native
from chunkflow_b200.lib import load_source

from .base import PatchInferencerBase

DEFAULT_MODEL_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "..", "convnet", "unet3l.py")
DEFAULT_MODEL_FILE = os.path.normpath(DEFAULT_MODEL_FILE)


def is_canonical_model(convnet_model) -> bool:
    """True if the model file is (or re-exports) the U-Net family the kernels implement (convnet/unet3l.py)."""
    if convnet_model is None:
        return True
    try:
        src = load_source(os.path.expanduser(convnet_model))
    except Exception:
        return False
    return hasattr(src, "LAYER_SPEC") and hasattr(src, "UNet3L")


def load_state_dict(convnet_model=None, convnet_weight_path=None) -> dict:
    """name -> float32 ndarray, through the model file's own loader (the same entry point the
    reference's ``-f pytorch`` uses, patch/pytorch.py:48-60) or from an ``.npz`` archive."""
    if convnet_weight_path and str(convnet_weight_path).endswith(".npz"):
        with np.load(convnet_weight_path) as z:
            return {k: z[k].astype(np.float32) for k in z.files}
    src = load_source(os.path.expanduser(convnet_model) if convnet_model else DEFAULT_MODEL_FILE)
    if hasattr(src, "load_model"):
        model = src.load_model(convnet_weight_path)
    else:
        import torch
        model = src.InstantiatedModel
        chkpt = torch.load(convnet_weight_path, map_location="cpu")
        model.load_state_dict(chkpt["state_dict"] if "state_dict" in chkpt else chkpt)
    return {k: v.detach().cpu().numpy().astype(np.float32) for k, v in model.state_dict().items()}


def precision_code(dtype: str = "float32", precision=None) -> int:
    """``--dtype`` -> precision mode of the convolution stack.

    float32 -> 'f16f8' (default): wgmma tensor cores, fp16 main product plus ONE e4m3 product of twice the K depth that
    carries both hi/lo correction terms, fp32 accumulation -- two tensor-core products per multiply (csrc/act_format.cuh);
    the tests assert <= 5e-4 max-abs against the fp32 CPU reference (the bar is 1e-3).
    'f16x3': fp16 hi/lo split operands, three products per multiply, asserted <= 2e-4.
    float16 -> 'f16': single-pass fp16 tensor cores, asserted <= 2e-2 (the reference documents float16 as a lower-precision
    option, flow.py:1871-1874).  ``precision`` (or env CHUNKFLOW_B200_PRECISION) forces one of 'simt' (fp32 FFMA on CUDA
    cores), 'f16x3', 'f16f8', 'f16'.
    """
    names = {"simt": _native.PRECISION_F32_SIMT, "f16x3": _native.PRECISION_F16X3_UMMA, "f16": _native.PRECISION_F16_UMMA,
             "f16f8": _native.PRECISION_F16F8_UMMA}
    precision = precision or os.environ.get("CHUNKFLOW_B200_PRECISION")
    if precision is not None:
        if isinstance(precision, int):
            return precision
        return names[str(precision).lower()]
    return DEFAULT_PRECISION[str(np.dtype(dtype))]


DEFAULT_PRECISION = {"float32": _native.PRECISION_F16F8_UMMA, "float16": _native.PRECISION_F16_UMMA}


class _DeviceBackend(PatchInferencerBase):
    framework = None

    def __init__(self, convnet_model, convnet_weight_path, input_patch_size, output_patch_size=None,
                 output_patch_overlap=None, num_output_channels: int = 1, dtype: str = "float32", bump: str = "wu",
                 batch_size: int = 1, device: int = 0, precision=None):
        assert bump == "wu"  # reference patch/pytorch.py:35
        if output_patch_size is None:
            output_patch_size = input_patch_size
        super().__init__(input_patch_size, output_patch_size, output_patch_overlap, num_output_channels, dtype=dtype)
        self.engine = _native.Engine(
            input_patch_size=self.input_patch_size, output_patch_size=self.output_patch_size,
            output_patch_overlap=self.output_patch_overlap, output_crop_margin=(0, 0, 0),
            num_output_channels=num_output_channels, batch_size=batch_size, framework=self.framework,
            precision=precision_code(dtype, precision), device=device)
        if self.framework == _native.FRAMEWORK_UNET3L:
            self.engine.load_state_dict(load_state_dict(convnet_model, convnet_weight_path))

    @property
    def compute_device(self) -> str:
        return self.engine.device_name

    def __call__(self, input_patch: np.ndarray) -> np.ndarray:
        input_patch = self._reshape_patch_to_5d(input_patch)
        assert input_patch.shape[1] == 1, "one input channel"
        return self.engine.patch_forward_host(input_patch.astype(np.float32, copy=False))


class B200(_DeviceBackend):
    framework = _native.FRAMEWORK_UNET3L


class Identity(_DeviceBackend):
    framework = _native.FRAMEWORK_IDENTITY

    def __init__(self, convnet_model=None, convnet_weight_path=None, input_patch_size=None, output_patch_overlap=None,
                 output_patch_size=None, num_output_channels: int = 1, dtype="float32", bump: str = "wu", **kw):
        super().__init__(convnet_model, convnet_weight_path, input_patch_size, output_patch_size,
                         output_patch_overlap, num_output_channels, dtype, bump, **kw)
