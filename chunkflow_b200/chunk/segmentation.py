"""A segmentation chunk (reference chunk/segmentation.py:17-109): ``Segmentation.evaluate`` scores it against ground truth,
``remap`` renumbers its ids, ``mask_fragments`` and ``mask_except`` remove dust and unselected objects.

Everything is computed on the GPU (``DeviceChunk.evaluate``, csrc/evaluate.cu; ``DeviceChunk.remap`` / ``mask_out_objects``,
csrc/relabel.cu): host chunks are uploaded for the call and the result is downloaded.  There is no CPU fallback.
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

    def remap(self, base_id: int = 0, device="cuda:0"):
        """renumber the object ID (reference chunk/segmentation.py:69-84)

        Args:
            base_id (int, optional): the maximum object ID in previous chunk. Defaults to 0.

        Returns:
            new_base_id (int): the maximum object ID in this chunk as the new base ID (0 for an all-zero chunk, whatever
            ``base_id``, like the reference).  ``self.array`` becomes uint64.
        """
        dev = _device_labels(self, device)
        new_base_id = dev.remap(base_id)
        self.array = dev.tensor.cpu().numpy().view(np.uint64)
        return np.uint64(new_base_id)

    def fill_holes(self, mode: str = "binary", return_fill_count: bool = False, device="cuda:0"):
        """A new Segmentation with the holes filled (DeviceChunk.fill_holes: ``binary`` is fill_voids.fill, ``keep-enclosed``
        and ``remove-enclosed`` fill per object), same dtype, offset and voxel size; with ``return_fill_count`` also the number
        of voxels the rule assigned.  Runs on the GPU."""
        from .device import DeviceChunk, _torch
        arr = np.ascontiguousarray(self.array)
        host = arr.view({4: np.int32, 8: np.int64}[arr.itemsize]) if arr.dtype in (np.uint32, np.uint64) else arr
        out, count = DeviceChunk(_torch().from_numpy(host).to(device)).fill_holes(mode, return_fill_count=True)
        seg = Segmentation(out.tensor.cpu().numpy().view(arr.dtype), voxel_offset=self.voxel_offset, voxel_size=self.voxel_size)
        return (seg, count) if return_fill_count else seg

    def mask_fragments(self, voxel_num_threshold: int, device="cuda:0"):
        """Ids with ``voxel count <= voxel_num_threshold`` become 0 (reference chunk/segmentation.py:86-90)."""
        mask_out_objects(self, dust_size_threshold=voxel_num_threshold, device=device)

    def mask_except(self, selected_obj_ids, device="cuda:0"):
        """Ids outside ``selected_obj_ids`` (a list, a set, "34,45,56" or a local .json file) become 0 (reference
        chunk/segmentation.py:92-109)."""
        if selected_obj_ids is None:
            print('we have not selected any objects to mask out.')
            return
        mask_out_objects(self, selected_obj_ids=selected_obj_ids, device=device)


def evaluate(segmentation, groundtruth, size_threshold: int = 1000, device="cuda:0") -> dict:
    """Segmentation.evaluate for any mix of host chunks, arrays and DeviceChunks (a DeviceChunk segmentation keeps its GPU);
    prints the reference's five lines and returns its dict."""
    seg = _device_labels(segmentation, device)
    gt = _device_labels(groundtruth, seg.tensor.device)
    ret = seg.evaluate(gt, size_threshold=size_threshold)
    print(report(ret), end="")
    return ret


def _host_labels(dev, dtype) -> np.ndarray:
    """The labels of a DeviceChunk made by _device_labels, back in the host dtype they came from."""
    arr = dev.tensor.cpu().numpy()
    if arr.dtype == np.int32:
        return arr.view(np.uint32).astype(dtype, copy=False)
    if arr.dtype == np.int64:
        return arr.view(np.uint64).astype(dtype, copy=False)   # masked values are 0 or unchanged: they fit
    return arr.astype(dtype, copy=False)


def mask_out_objects(segmentation, dust_size_threshold=None, selected_obj_ids=None, device="cuda:0"):
    """``mask_fragments`` and then ``mask_except`` (the body of `mask-out-objects`, reference flow/flow.py:2044-2047) with
    one count pass and one relabelling pass on the GPU for both; prints the line mask_fragments prints.  A DeviceChunk is
    changed in place and stays on its GPU; a host chunk gets a new ``array`` of the same dtype.  Returns ``segmentation``."""
    from .device import DeviceChunk
    dev = _device_labels(segmentation, device)
    report = dev.mask_out_objects(dust_size_threshold, selected_obj_ids)
    if report is not None and dust_size_threshold is not None:
        num, dust = report
        print(f'masking out {dust} fragments in {num} with a percentage of {dust / num}')   # reference segmentation.py:89
    if report is not None and not isinstance(segmentation, DeviceChunk):
        segmentation.array = _host_labels(dev, segmentation.array.dtype)
    return segmentation
