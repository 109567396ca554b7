"""Chunk-level overlap-tile convnet inference on an H100.

Drop-in for the reference's ``Inferencer``
(chunkflow/flow/divid_conquer/inferencer.py:21-479): same constructor keywords, same
``__call__(Chunk) -> Chunk``, same ``compute_device`` / context-manager surface -- but the
chunk is uploaded once, every patch is extracted, run through the network, bump-weighted
and blended by CUDA kernels on the device, and the normalised result is downloaded once.

Frameworks:
  'b200'      the plain U-Net family of depth 2 to 4 (chunkflow_b200/convnet/unet3l.py) as sm_90a kernels.
  'pytorch'   accepted when the model file is that canonical U-Net (the same file drives the
              reference's ``-f pytorch`` CPU path, the parity oracle); any other torch model
              is refused -- there is no CPU / eager fallback.
  'identity'  reference patch/identity.py on the device (known-answer tests).
  'universal' / 'prebuilt'  user-supplied per-patch backends (host numpy in/out); extract,
              blend and normalise still run on the device.
"""
from __future__ import annotations

import os
import sys
from typing import Union
from warnings import warn

import numpy as np

from chunkflow_b200 import _native
from chunkflow_b200.chunk import Chunk
from chunkflow_b200.lib.cartesian_coordinate import Cartesian, to_cartesian

from .patch.base import PatchInferencerBase
from .patch import b200 as b200_patch
from .transform import TransformSequences


class Inferencer(object):
    def __init__(self,
                 convnet_model: Union[str, PatchInferencerBase, None],
                 convnet_weight_path: Union[str, None],
                 input_patch_size: Union[tuple, list, Cartesian],
                 output_patch_size: Union[tuple, list, Cartesian] = None,
                 patch_num: Union[tuple, list, Cartesian] = None,
                 num_input_channels: int = 1,
                 num_output_channels: int = 3,
                 output_patch_overlap: Union[tuple, list, Cartesian] = None,
                 output_crop_margin: Union[tuple, list, Cartesian] = None,
                 dtype='float32',
                 framework: str = 'universal',
                 batch_size: int = 1,
                 bump: str = 'wu',
                 input_size: Union[tuple, list, Cartesian] = None,
                 mask_output_chunk: bool = True,
                 mask_myelin_threshold=None,
                 augment: Union[bool, str] = False,
                 dry_run: bool = False,
                 device: int = None,
                 precision=None):
        assert input_size is None or patch_num is None
        assert bump == 'wu', 'only the wu bump function is supported (reference patch/pytorch.py:35)'

        input_patch_size = to_cartesian(input_patch_size)
        patch_num = to_cartesian(patch_num)
        input_size = to_cartesian(input_size)
        output_patch_size = to_cartesian(output_patch_size)
        output_patch_overlap = to_cartesian(output_patch_overlap)
        output_crop_margin = to_cartesian(output_crop_margin)

        if output_patch_size is None:
            output_patch_size = input_patch_size
        if output_patch_overlap is None:
            output_patch_overlap = output_patch_size // 2

        self.input_patch_size = input_patch_size
        self.output_patch_size = output_patch_size
        self.output_patch_overlap = output_patch_overlap
        self.patch_num = patch_num
        self.batch_size = batch_size
        self.input_size = input_size

        # reference inferencer.py:98-107
        if output_crop_margin is None:
            self.output_crop_margin = Cartesian(0, 0, 0) if mask_output_chunk else self.output_patch_overlap
        else:
            self.output_crop_margin = output_crop_margin
            # the overlap region is reweighted by the patch mask: always crop at least that much
            assert self.output_crop_margin >= self.output_patch_overlap

        # reference inferencer.py:109-122
        self.output_patch_crop_margin = (input_patch_size - output_patch_size) // 2
        self.output_offset = self.output_crop_margin
        self.output_patch_stride = tuple(s - o for s, o in zip(output_patch_size, output_patch_overlap))
        self.input_patch_overlap = tuple(
            c * 2 + o for c, o in zip(self.output_patch_crop_margin, self.output_patch_overlap))
        self.input_patch_stride = tuple(p - o for p, o in zip(input_patch_size, self.input_patch_overlap))

        if not mask_output_chunk:
            # no chunk-wise mask: the patches must tile the chunk exactly (reference :125-139)
            assert (self.input_size is not None) or (self.patch_num is not None)
            if patch_num is None:
                self.patch_num = tuple((isz - o) // s for isz, o, s in zip(
                    self.input_size, self.input_patch_overlap, self.input_patch_stride))
            if self.input_size is None:
                self.input_size = tuple(pst * pn + po for pst, pn, po in zip(
                    self.input_patch_stride, self.patch_num, self.input_patch_overlap))
            self.output_size = tuple(pst * pn + po - 2 * ocm for pst, pn, po, ocm in zip(
                self.output_patch_stride, self.patch_num, self.output_patch_overlap, self.output_crop_margin))
        else:
            self.input_size = None
            self.output_size = None

        self.num_input_channels = num_input_channels
        self.num_output_channels = num_output_channels
        self.mask_output_chunk = mask_output_chunk
        self.dtype = dtype
        self.mask_myelin_threshold = mask_myelin_threshold
        self.dry_run = dry_run
        self.framework = framework
        self.patch_slices_list = []
        self.timing = {}

        if device is None:
            device = int(os.environ.get('LOCAL_RANK', 0))
        self.device = device

        if isinstance(convnet_model, str):
            convnet_model = os.path.expanduser(convnet_model)
        if isinstance(convnet_weight_path, str):
            convnet_weight_path = os.path.expanduser(convnet_weight_path)

        # augment: False | True (= 'reference': the reference's arithmetic, literally -- its flips act on the channel /
        # batch axes, transform.py:30-52) | 'spatial' (the intended spatial flips; explicit opt-in, different numbers)
        self.augment = _native.augment_code(augment)
        self.transform_sequences = None
        if self.augment:
            self.transform_sequences = TransformSequences(
                'spatial' if self.augment == _native.AUGMENT_SPATIAL else 'reference')
        self._prepare_patch_inferencer(framework, convnet_model, convnet_weight_path, bump, precision)

    # ------------------------------------------------------------------------------------
    def _engine(self, framework_code, precision=None, augment=0):
        return _native.Engine(
            input_patch_size=self.input_patch_size,
            # a host plugin returns cropped patches: to the device they are crop-free patches
            output_patch_size=self.output_patch_size,
            output_patch_overlap=self.output_patch_overlap,
            output_crop_margin=self.output_crop_margin,
            num_input_channels=self.num_input_channels,
            num_output_channels=self.num_output_channels,
            batch_size=self._patches_in_flight(framework_code),
            mask_output_chunk=self.mask_output_chunk,
            framework=framework_code,
            precision=b200_patch.precision_code(self.dtype, precision),
            device=self.device,
            mask_myelin_threshold=self.mask_myelin_threshold,
            augment=augment,
            check_output_range=True)

    def _patches_in_flight(self, framework_code) -> int:
        """``batch_size`` is a scheduling hint here (the reference asserts 1 for pytorch although its examples pass
        12, inferencer.py:216-220).  With the default of 1 the device network path picks the number of patches in
        flight itself: enough CTAs to fill 132 SMs at every U-Net level, bounded by a quarter of the free memory at
        600 bytes per patch voxel: the activations of the default f16f8 mode take about 552 bytes per patch voxel at
        depth 3 and about 620 at depth 4 (the 4-level network may hold a few percent more than the quarter)."""
        if self.batch_size > 1 or framework_code != _native.FRAMEWORK_UNET3L:
            return self.batch_size
        free, _ = _native.device_memory(self.device)
        per_patch = int(np.prod(self.input_patch_size)) * 600
        return int(max(1, min(12, (free // 4) // max(per_patch, 1))))

    def _prepare_patch_inferencer(self, framework, convnet_model, convnet_weight_path, bump, precision):
        self.patch_inferencer = None   # host-side per-patch plugin (universal / prebuilt) if any
        if framework == 'pytorch' and not b200_patch.is_canonical_model(convnet_model):
            raise NotImplementedError(
                "framework='pytorch' is served by hand-written kernels for the plain U-Net family of depth 2 to 4 "
                "(chunkflow_b200/convnet/unet3l.py) only; arbitrary torch models have no CPU/eager fallback here. "
                "Wrap other backends as a `universal` plugin.")
        if framework in ('b200', 'pytorch'):
            # --augment on the device: the variants of a patch are extra batch entries, averaged by the blend
            # (reference-literal by default, 'spatial' on request; include/chunkflow_b200.h CFB_AUGMENT_*)
            self.engine = self._engine(_native.FRAMEWORK_UNET3L, precision, augment=self.augment)
            self.engine.load_state_dict(b200_patch.load_state_dict(convnet_model, convnet_weight_path))
        elif framework == 'identity':
            if self.transform_sequences is not None:
                # identity o (transform, inverse transform) == identity: run the plugin-level path so
                # that the augmentation code is exercised exactly like the reference test does
                self.patch_inferencer = b200_patch.Identity(
                    None, None, self.input_patch_size, self.output_patch_overlap, self.output_patch_size,
                    self.num_output_channels, self.dtype, bump, batch_size=self.batch_size, device=self.device)
            self.engine = self._engine(_native.FRAMEWORK_IDENTITY)
        elif framework == 'prebuilt':
            self.patch_inferencer = convnet_model
            self.engine = self._engine(_native.FRAMEWORK_IDENTITY)
        elif framework == 'universal':
            from .patch.universal import Universal
            self.patch_inferencer = Universal(
                convnet_model, convnet_weight_path,
                input_patch_size=self.input_patch_size, output_patch_size=self.output_patch_size,
                output_patch_overlap=self.output_patch_overlap, num_output_channels=self.num_output_channels,
                dtype=self.dtype, bump=bump)
            self.engine = self._engine(_native.FRAMEWORK_IDENTITY)
        else:
            raise Exception(f'invalid inference backend: {framework}')
        self.input_patch_buffer = None
        if self.patch_inferencer is not None and self.transform_sequences is not None:
            # the transposed patch is fed to the same backend: it must have the same shape (the reference fails
            # inside numpy / the backend here)
            if self.input_patch_size[1] != self.input_patch_size[2] or self.output_patch_size[1] != self.output_patch_size[2]:
                raise ValueError('--augment transposes y and x: the patch must be square in y, x')
        if self.patch_inferencer is not None:
            # reused host staging buffer, like the reference (inferencer.py:154-155)
            self.input_patch_buffer = np.zeros(
                (self.batch_size, self.num_input_channels, *self.input_patch_size), dtype=np.float32)

    @property
    def compute_device(self):
        if self.patch_inferencer is not None and hasattr(self.patch_inferencer, 'compute_device'):
            try:
                return self.patch_inferencer.compute_device
            except Exception:
                pass
        return self.engine.device_name

    def __enter__(self):
        return self

    def __exit__(self, exception_type, exception_value, traceback):
        pass

    # ------------------------------------------------------------------------------------
    def _check_alignment(self):
        is_align = tuple((i - o) % s == 0 for i, s, o in zip(
            self.input_size[-3:], self.input_patch_stride, self.input_patch_overlap))
        # without the chunk-wise mask every axis must be tiled exactly (reference :243-253)
        assert np.all(is_align), 'the patches do not align with the input chunk'

    def _update_parameters_for_input_chunk(self, input_chunk: Chunk):
        if self.input_size is not None and tuple(self.input_size[-3:]) != tuple(input_chunk.shape[-3:]):
            warn('the input size has changed, using new intput size.')
        self.input_size = tuple(input_chunk.shape[-3:])
        if not self.mask_output_chunk:
            self._check_alignment()
        self.output_size = (self.num_output_channels,) + tuple(
            isz - 2 * oc for isz, oc in zip(self.input_size, self.output_offset))
        self._construct_patch_slices_list(input_chunk.voxel_offset)

    def _construct_patch_slices_list(self, input_chunk_offset):
        """(input slices, output slices) per patch in GLOBAL coordinates; z-major then y then x, the
        last patch per axis clamped back into the chunk (reference inferencer.py:255-292).  The
        start grid comes from the native library -- the same table the kernels iterate."""
        starts = self.engine.patch_grid(self.input_size)
        off = tuple(input_chunk_offset)
        cm = self.output_patch_crop_margin
        self.patch_slices_list = []
        for s in starts:
            gi = tuple(int(a) + o for a, o in zip(s, off))
            go = tuple(g + c for g, c in zip(gi, cm))
            self.patch_slices_list.append((
                tuple(slice(g, g + p) for g, p in zip(gi, self.input_patch_size)),
                tuple(slice(g, g + p) for g, p in zip(go, self.output_patch_size))))

    def _prepare_input_array(self, input_chunk: Chunk) -> np.ndarray:
        arr = input_chunk.array
        if arr.ndim == 4:
            assert arr.shape[0] == 1, 'one input channel'
            arr = arr[0]
        if arr.dtype == np.uint8 or arr.dtype == np.float32:
            return arr
        if np.issubdtype(arr.dtype, np.integer):
            # wider integers: normalise to [0,1] by the dtype maximum like the reference (:395-399)
            return (arr.astype(np.float32) / np.float32(np.iinfo(arr.dtype).max)).astype(np.float32)
        return arr.astype(np.float32)

    def __call__(self, input_chunk: Chunk, output_buffer: np.ndarray = None) -> Chunk:
        """``output_buffer`` (optional extension): a preallocated C-contiguous float32 array of the
        output shape, e.g. a view of pinned host memory, that receives the result."""
        assert isinstance(input_chunk, Chunk)
        self._update_parameters_for_input_chunk(input_chunk)
        output_voxel_offset = tuple(io + oc for io, oc in zip(input_chunk.voxel_offset, self.output_offset))

        if self.dry_run:
            print('dry run, return a special artifical chunk.')
            size = self.output_size
            if self.mask_myelin_threshold:
                size = (size[0] - 1, *size[1:])
            return Chunk.create(size=size, dtype=np.dtype('float32'), voxel_offset=output_voxel_offset,
                                voxel_size=input_chunk.voxel_size)

        arr = self._prepare_input_array(input_chunk)
        if output_buffer is not None:
            assert output_buffer.shape == tuple(self.output_size) and output_buffer.dtype == np.float32
            out = output_buffer
        else:
            out = self._result_array(self.output_size)
        try:
            if self.patch_inferencer is None:
                self.engine.infer_chunk_host(arr, out)
                self.timing = self.engine.last_timing()
            else:
                self._run_host_plugin(arr, out)
        except _native.NativeError as err:
            if err.code == _native.ERR_OUTPUT_RANGE:
                # the reference raises AssertionError here (inferencer.py:465-466)
                raise AssertionError('output buffer should not be greater than 1') from err
            raise

        if self.mask_myelin_threshold:
            assert out.shape[0] == 4
            out = out[:-1]
        return Chunk(out, voxel_offset=output_voxel_offset, voxel_size=input_chunk.voxel_size)

    def _result_array(self, shape) -> np.ndarray:
        """A float32 array for the result chunk (the reference allocates one per call, inferencer.py:190-198).  A 1024^3
        result is 12.9 GB = 3.1 million pages: inside a VM the first touch and above all the later ``munmap`` of that many
        pages cost seconds (measured 1.6 s for the free alone, more with huge pages).  The last result array is therefore
        kept and handed out AGAIN once the caller has dropped every reference to it (views and buffer exports hold
        references, so a result that is still in use is never recycled); otherwise a new array is allocated."""
        shape = tuple(int(v) for v in shape)
        buf = getattr(self, '_last_result', None)
        if buf is not None and buf.shape == shape and sys.getrefcount(buf) <= 3:  # self._last_result, buf, getrefcount's argument
            return buf
        buf = None
        self._last_result = None           # release the old one before allocating (peak memory)
        out = np.empty(shape, dtype=np.float32)
        if out.nbytes >= (64 << 20):
            self._last_result = out
        return out

    def infer_device(self, input_chunk):
        """Extension (SURVEY section 8 f3): the same operator on a :class:`chunkflow_b200.chunk.device.DeviceChunk` --
        uint8 (or float32 in [0,1]) image already in GPU memory in, float32 affinity map in GPU memory out, nothing
        crosses PCIe.  Built-in device backends only (``b200`` / ``identity``)."""
        import torch
        from chunkflow_b200.chunk.device import DeviceChunk
        assert isinstance(input_chunk, DeviceChunk)
        assert self.patch_inferencer is None, 'infer_device needs a built-in device backend (framework b200 / identity)'
        t = input_chunk.tensor
        if t.ndim == 4:
            assert t.shape[0] == 1, 'one input channel'
            t = t[0]
        assert t.dtype in (torch.uint8, torch.float32)
        assert t.device.index == self.engine.params.device, 'the chunk must live on the engine\'s GPU'
        self._update_parameters_for_input_chunk(input_chunk)
        output_voxel_offset = tuple(io + oc for io, oc in zip(input_chunk.voxel_offset, self.output_offset))
        out = torch.empty(self.output_size, dtype=torch.float32, device=t.device)
        try:
            with torch.cuda.device(t.device):
                stream = torch.cuda.current_stream(t.device)
                self.engine.infer_chunk_device(t.data_ptr(), np.uint8 if t.dtype == torch.uint8 else np.float32,
                                               tuple(t.shape), out.data_ptr(), stream.cuda_stream)
                stream.synchronize()  # the range check of the result is reported by the call above
            self.timing = self.engine.last_timing()
        except _native.NativeError as err:
            if err.code == _native.ERR_OUTPUT_RANGE:
                raise AssertionError('output buffer should not be greater than 1') from err
            raise
        if self.mask_myelin_threshold:
            assert out.shape[0] == 4
            out = out[:-1]
        return DeviceChunk(out, voxel_offset=output_voxel_offset, voxel_size=input_chunk.voxel_size)

    def _run_host_plugin(self, arr: np.ndarray, out: np.ndarray) -> None:
        """universal / prebuilt backends: device extract -> host callable -> device blend."""
        eng = self.engine
        eng.plugin_begin(arr)
        n = len(self.patch_slices_list)
        for i in range(0, n, self.batch_size):
            nb = min(self.batch_size, n - i)
            # stale slots of the last partial batch are computed and dropped, like the reference (:408-411,436)
            eng.plugin_extract(i, nb, self.input_patch_buffer[:nb])
            if self.transform_sequences is None:
                output_patch = self.patch_inferencer(self.input_patch_buffer)
            else:
                patches = self.transform_sequences.forward(self.input_patch_buffer)
                outs = [self.patch_inferencer(p) for p in patches]
                outs = self.transform_sequences.backward(outs)
                output_patch = sum(outs) / len(outs)
            assert isinstance(output_patch, np.ndarray)
            eng.plugin_blend(i, nb, output_patch[:nb, :self.num_output_channels])
        eng.plugin_end(out)
