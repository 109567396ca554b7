"""Fill the holes of a segmentation -- drop-in for the reference's plugin ``chunkflow/plugins/fill_segmentation_holes.py``, which
returns ``[Chunk(fill_voids.fill(seg.array))]`` with the input's properties.

Same signature and return value.  The holes are found on the GPU (``csrc/fill_holes.cu``, rules in
``oracle/fill_holes_oracle.py``: fill_voids is not vendored, its output is restated): every voxel != 0 and every background
voxel with no 6-connected background path to outside the chunk becomes 1, every other voxel 0, in the input's dtype.  A host
``Chunk`` goes to the GPU for the call and comes back as a ``Chunk``; a ``DeviceChunk`` is read where it is.  There is no CPU
fallback.
"""
from chunkflow_b200.chunk import Chunk


def execute(seg: Chunk):
    from chunkflow_b200.chunk.device import DeviceChunk
    dev = seg if isinstance(seg, DeviceChunk) else DeviceChunk.from_chunk(seg)
    array = dev.fill_holes("binary").tensor.cpu().numpy()
    seg2 = Chunk(array, voxel_offset=seg.voxel_offset, voxel_size=seg.voxel_size,
                 layer_type=seg.layer_type if isinstance(seg, DeviceChunk) else seg._layer_type)
    return [seg2, ]
