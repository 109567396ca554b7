"""Host-side ``Chunk`` container: an ndarray plus its place in the big volume.

Only the surface the ``inference`` hot path touches is provided (SURVEY.md section 8a
rows a7, a11, a12, a14, a16, a17); file I/O, meshing, evaluation etc. are out of scope.
Reference: chunkflow/chunk/base.py:28 (``class Chunk``).

Differences from the reference that are deliberate:

* ``layer_type`` is guessed lazily (the reference scans min/max of the whole array in
  every constructor call, base.py:78-91,510-514 -- 4 % of its non-network time).
* ``create(pattern='random')`` for integer dtypes returns plain random integers; the
  reference relabels them with connected components (base.py:191-193), which makes
  them unusable as uint8 images.
"""
from __future__ import annotations

from numbers import Number
from typing import Optional, Sequence, Tuple, Union

import numpy as np
from numpy.lib.mixins import NDArrayOperatorsMixin

from chunkflow_b200.lib.cartesian_coordinate import Cartesian

_LAYER_TYPES = (None, "image", "segmentation", "probability_map", "affinity_map", "unknown")


class Chunk(NDArrayOperatorsMixin):
    _HANDLED_TYPES = (np.ndarray, Number)

    def __init__(self, array, voxel_offset=None, voxel_size=None, layer_type: Optional[str] = None):
        if isinstance(array, Chunk):
            if voxel_offset is None:
                voxel_offset = array.voxel_offset
            array = array.array
        if not isinstance(array, np.ndarray):
            raise TypeError("Chunk wraps a numpy.ndarray")
        if array.ndim == 2:
            array = array[np.newaxis]
        if array.ndim not in (3, 4):
            raise ValueError(f"Chunk array must be 3-D (zyx) or 4-D (czyx), got {array.ndim}-D")
        if layer_type not in _LAYER_TYPES:
            raise ValueError(f"layer type: {layer_type} is unsupported!")
        self.array = array

        if voxel_offset is None:
            voxel_offset = (0, 0, 0)
        voxel_offset = tuple(voxel_offset)
        if len(voxel_offset) == 4:
            if voxel_offset[0] != 0:
                raise ValueError("the channel component of a 4-D voxel offset must be 0")
            voxel_offset = voxel_offset[1:]
        self.voxel_offset = Cartesian.from_collection(voxel_offset)

        if voxel_size is not None:
            voxel_size = Cartesian.from_collection(tuple(voxel_size))
            if not all(v > 0 for v in voxel_size):
                raise ValueError("voxel size must be positive")
        self.voxel_size = voxel_size
        self._layer_type = layer_type

    # ---- constructors --------------------------------------------------------------
    @classmethod
    def create(cls, size=(64, 64, 64), dtype=np.uint8, voxel_offset=(0, 0, 0),
               voxel_size=None, pattern: str = "sin", high: int = 255, seed: Optional[int] = None):
        """Synthetic chunk (reference: base.py:139-199).

        ``pattern='sin'`` is ``abs(sin(4 (i_z + i_y + i_x)))`` with ``i = linspace(0,1,n)``
        (base.py:170-179): deterministic, the input of BASELINE config #1.
        """
        dtype = np.dtype(dtype)
        size = tuple(size)
        if pattern == "zero":
            arr = np.zeros(size, dtype=dtype)
        elif pattern == "sin":
            grids = np.meshgrid(*[np.linspace(0, 1, n) for n in size[-3:]], indexing="ij")
            arr = np.abs(np.sin(4 * (grids[0] + grids[1] + grids[2])))
            if len(size) == 4:
                arr = np.repeat(arr[np.newaxis], size[0], axis=0)
            if dtype == np.uint8:
                arr = (arr * 255).astype(dtype)
            elif np.issubdtype(dtype, np.floating):
                arr = arr.astype(dtype)
            else:
                raise NotImplementedError(f"do not support this data type: {dtype}")
        elif pattern == "random":
            rng = np.random.default_rng(seed)
            if np.issubdtype(dtype, np.floating):
                arr = rng.random(size).astype(dtype)
            elif np.issubdtype(dtype, np.integer):
                arr = rng.integers(0, high, size=size, dtype=dtype)
            else:
                raise NotImplementedError(f"do not support this data type: {dtype}")
        else:
            raise NotImplementedError(f"do not support the pattern: {pattern}")
        return cls(arr, voxel_offset=voxel_offset, voxel_size=voxel_size)

    # ---- array protocol ------------------------------------------------------------
    def __array__(self, dtype=None, copy=None):
        return self.array if dtype is None else self.array.astype(dtype, copy=False)

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        """numpy dispatch so that ``chunk *= mask_chunk`` works (reference base.py:418-453)."""
        out = kwargs.get("out", ())
        for x in inputs + out:
            if not isinstance(x, self._HANDLED_TYPES + (Chunk,)):
                return NotImplemented
        inputs = tuple(x.array if isinstance(x, Chunk) else x for x in inputs)
        if out:
            kwargs["out"] = tuple(x.array if isinstance(x, Chunk) else x for x in out)
        result = getattr(ufunc, method)(*inputs, **kwargs)
        if isinstance(result, tuple):
            return tuple(self._like(r) for r in result)
        if method == "at":
            return None
        if isinstance(result, np.ndarray) and result.ndim >= 3:
            return self._like(result)
        return result

    def _like(self, array):
        return Chunk(array, voxel_offset=self.voxel_offset, voxel_size=self.voxel_size)

    def __getitem__(self, index):
        return self.array[index]

    def __setitem__(self, key, value):
        self.array[key] = value

    def __len__(self):
        return len(self.array)

    # ---- geometry ------------------------------------------------------------------
    @property
    def shape(self) -> tuple:
        return self.array.shape

    @property
    def ndim(self) -> int:
        return self.array.ndim

    @property
    def dtype(self) -> np.dtype:
        return self.array.dtype

    @property
    def size(self) -> int:
        return self.array.size

    @property
    def ndoffset(self) -> tuple:
        """voxel offset padded to the array rank (reference base.py:559-566)."""
        off = tuple(self.voxel_offset)
        return (0,) + off if self.ndim == 4 else off

    @property
    def slices(self) -> tuple:
        return tuple(slice(o, o + s) for o, s in zip(self.ndoffset, self.shape))

    @property
    def voxel_stop(self) -> tuple:
        return tuple(o + s for o, s in zip(self.ndoffset, self.shape))

    @property
    def is_image(self) -> bool:
        """uint8 and 3-D (reference chunk/base.py:495-497)."""
        return self.array.dtype == np.uint8 and self.array.ndim == 3

    # ---- layer type guess (lazy) ---------------------------------------------------
    @property
    def layer_type(self) -> str:
        if self._layer_type is None:
            a = self.array
            if a.ndim == 3 and a.dtype == np.uint8:
                self._layer_type = "image"
            elif a.ndim == 3 and (np.issubdtype(a.dtype, np.integer) or a.dtype == bool):
                self._layer_type = "segmentation"
            elif a.dtype == np.float32 and a.size and a.max() <= 1.0 and a.min() >= 0.0:
                # 'probability_map' wins over 'affinity_map' like the reference (base.py:86-89)
                self._layer_type = "probability_map"
            elif a.ndim == 4 and a.shape[0] == 3 and a.dtype == np.float32:
                self._layer_type = "affinity_map"
            else:
                self._layer_type = "unknown"
        return self._layer_type

    @layer_type.setter
    def layer_type(self, value):
        if value not in _LAYER_TYPES:
            raise ValueError(f"layer type: {value} is unsupported!")
        self._layer_type = value

    # ---- hot-path operations -------------------------------------------------------
    def astype(self, dtype):
        if dtype is None or np.dtype(dtype) == self.array.dtype:
            return self
        return self._like(self.array.astype(dtype))

    def cutout(self, slices: Sequence[slice]) -> "Chunk":
        """Sub-box given in GLOBAL voxel slices (reference base.py:761-781)."""
        slices = tuple(slices)
        if len(slices) == self.ndim - 1:
            slices = (slice(0, self.shape[0]),) + slices
        if len(slices) != self.ndim:
            raise ValueError("cutout slices do not match the chunk rank")
        local = tuple(slice(s.start - o, s.stop - o) for s, o in zip(slices, self.ndoffset))
        for s, n in zip(local, self.shape):
            if s.start < 0 or s.stop > n:
                raise IndexError("cutout region is outside of the chunk")
        return Chunk(self.array[local], voxel_offset=tuple(s.start for s in slices[-3:]),
                     voxel_size=self.voxel_size, layer_type=self._layer_type)

    def blend(self, patch: "Chunk") -> None:
        """``self[box] += patch[clipped box]`` -- the patch box is clipped to this chunk
        (reference base.py:792-807)."""
        pslices = patch.slices
        if patch.ndim == self.ndim - 1:
            pslices = (slice(0, self.shape[0]),) + pslices
        dst, src = [], []
        for ps, o, n in zip(pslices, self.ndoffset, self.shape):
            lo, hi = max(ps.start - o, 0), min(ps.stop - o, n)
            dst.append(slice(lo, hi))
            src.append(slice(lo + o - ps.start, hi + o - ps.start))
        if patch.ndim == self.ndim - 1:
            src = src[1:]
        self.array[tuple(dst)] += patch.array[tuple(src)]

    def connected_component(self, threshold: float = None, connectivity: int = 6) -> "Chunk":
        """Threshold the map chunk and get connected components (reference chunk/base.py:128-137; cc3d's labelling runs as
        CUDA kernels: the chunk is moved to the GPU and back, there is no CPU fallback)."""
        from .device import DeviceChunk
        dev = DeviceChunk.from_chunk(self)
        return dev.connected_component(threshold=threshold, connectivity=connectivity).to_chunk()

    def gaussian_filter_2d(self, sigma=1, device="cuda:0") -> None:
        """Gaussian blur of every z section in place (reference chunk/base.py:846-853: ``gaussian_filter(array[..., z, :, :],
        sigma)`` for every z), bit-identical to scipy.ndimage.  On a (c,z,y,x) chunk the section is the (c,y,x) block, so the
        blur also runs across the channels, as in the reference.  It runs on the GPU (DeviceChunk.gaussian_filter_2d) and the
        result is written back into this chunk's array, so views of it see the change; there is no CPU fallback."""
        from .device import DeviceChunk
        dev = DeviceChunk.from_chunk(self, device=device)
        dev.gaussian_filter_2d(sigma)
        self.array[...] = dev.tensor.cpu().numpy()

    def mask_using_last_channel(self, threshold: float = 0.3) -> "Chunk":
        """Drop the last channel and zero where it is >= threshold (reference base.py:685-689)."""
        keep = self.array[-1] < threshold
        ret = self.array[:-1]
        ret *= keep
        return self._like(ret)

    def crop_margin(self, margin_size: Sequence[int]) -> "Chunk":
        mz, my, mx = margin_size
        sz, sy, sx = self.shape[-3:]
        arr = self.array[..., mz:sz - mz, my:sy - my, mx:sx - mx]
        return Chunk(arr, voxel_offset=self.voxel_offset + Cartesian(mz, my, mx), voxel_size=self.voxel_size)

    def __repr__(self):
        return (f"Chunk(shape={self.shape}, dtype={self.dtype}, voxel_offset={tuple(self.voxel_offset)}, "
                f"voxel_size={None if self.voxel_size is None else tuple(self.voxel_size)})")
