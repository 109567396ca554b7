"""A segmentation chunk (reference chunk/segmentation.py:17-67): ``Segmentation.evaluate`` scores it against ground truth.

The scores are computed on the GPU (``DeviceChunk.evaluate``, csrc/evaluate.cu): host chunks are uploaded for the call.
There is no CPU fallback.
"""
from __future__ import annotations

import numpy as np

from .base import Chunk


def _device_labels(chunk, device):
    """A DeviceChunk holding ``chunk``'s labels in a dtype the kernels read without changing any score: uint8 and uint32
    as they are, uint64 as its int64 bit pattern, any other integer type as ``astype(np.uint64)`` (what the reference does,
    segmentation.py:39-45).  A DeviceChunk is used as it is."""
    from .device import DeviceChunk, _torch
    if isinstance(chunk, DeviceChunk):
        return chunk
    arr = np.asarray(chunk.array if isinstance(chunk, Chunk) else chunk)
    if not np.issubdtype(arr.dtype, np.integer) and arr.dtype != np.bool_:
        raise TypeError(f"a segmentation has integer labels, not {arr.dtype}")
    if arr.dtype in (np.dtype(np.uint8), np.dtype(np.bool_)):
        host = np.ascontiguousarray(arr).view(np.uint8)
    elif arr.dtype == np.uint32:
        host = np.ascontiguousarray(arr).view(np.int32)
    else:
        host = np.ascontiguousarray(arr.astype(np.uint64, copy=False)).view(np.int64)
    torch = _torch()
    return DeviceChunk(torch.from_numpy(host).to(device), voxel_offset=getattr(chunk, "voxel_offset", None),
                       voxel_size=getattr(chunk, "voxel_size", None), layer_type="segmentation")


def report(scores: dict) -> str:
    """The five lines Segmentation.evaluate prints (reference segmentation.py:55-59)."""
    return (f"rand index: {scores['rand_index']: .3f}\n"
            f"adjusted rand index: {scores['adjusted_rand_index']: .3f}\n"
            f"variation of information: {scores['variation_of_information']: .3f}\n"
            f"edit distance: {scores['edit_distance']}\n"
            f"Fowlkes Mallows Index: {scores['fowlkes_mallows_index']: .3f}\n")


class Segmentation(Chunk):
    """A chunk of a segmentation volume: 3-D, integer labels (reference chunk/segmentation.py:17-24)."""

    def __init__(self, array, **kwargs):
        super().__init__(array, **kwargs)
        assert self.array.ndim == 3
        assert np.issubdtype(self.array.dtype, np.integer)

    @classmethod
    def from_chunk(cls, chunk):
        assert isinstance(chunk, Chunk)
        return cls(chunk.array, voxel_offset=chunk.voxel_offset, voxel_size=chunk.voxel_size)

    def evaluate(self, groundtruth, size_threshold: int = 1000, device="cuda:0") -> dict:
        """Scores against ``groundtruth`` (a Chunk, an array or a DeviceChunk of the same shape), printed and returned like
        the reference's: {'rand_index', 'adjusted_rand_index', 'variation_of_information', 'fowlkes_mallows_index',
        'edit_distance'}, edit distance = (false merges, false splits).

        Parameters:
            size_threshold [int]: size threshold for Edit Distance.
                Ignore splits or merges smaller than this number of voxels.
        """
        return evaluate(self, groundtruth, size_threshold, device)


def evaluate(segmentation, groundtruth, size_threshold: int = 1000, device="cuda:0") -> dict:
    """Segmentation.evaluate for any mix of host chunks, arrays and DeviceChunks (a DeviceChunk segmentation keeps its GPU);
    prints the reference's five lines and returns its dict."""
    seg = _device_labels(segmentation, device)
    gt = _device_labels(groundtruth, seg.tensor.device)
    ret = seg.evaluate(gt, size_threshold=size_threshold)
    print(report(ret), end="")
    return ret
