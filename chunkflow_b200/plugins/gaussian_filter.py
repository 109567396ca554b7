"""2-D Gaussian blur of every section -- drop-in for the reference's plugin ``chunkflow/plugins/gaussian_filter.py``
(``execute``, lines 7-23), which calls ``scipy.ndimage.gaussian_filter`` on every (channel,) z plane.

Same signature, same return value (the chunk, a clone unless ``inplace``), bit-identical to scipy.  Unlike the
``gaussian-filter`` command, a (c, z, y, x) chunk is filtered channel by channel.  The planes are filtered by CUDA kernels
(``csrc/filter_kernels.cuh``); a host ``Chunk`` goes to the GPU and back, a ``DeviceChunk`` stays there.  There is no CPU
fallback.
"""
import numpy as np

from chunkflow_b200.chunk import Chunk


def execute(chunk: Chunk, sigma: float = 1., inplace=False):
    from chunkflow_b200.chunk.device import DeviceChunk
    ndim = len(chunk.shape)
    if ndim not in (3, 4):
        raise ValueError(f'only support 4 or 3d, but got {ndim}')
    if isinstance(chunk, DeviceChunk):
        if not inplace:
            chunk = DeviceChunk(chunk.tensor.clone(), voxel_offset=chunk.voxel_offset, voxel_size=chunk.voxel_size,
                                layer_type=chunk.layer_type)
        chunk.gaussian_filter_2d(sigma, per_channel=True)
        return chunk
    if not inplace:
        chunk = Chunk(np.array(chunk.array, copy=True), voxel_offset=chunk.voxel_offset, voxel_size=chunk.voxel_size,
                      layer_type=chunk._layer_type)
    dev = DeviceChunk.from_chunk(chunk)
    dev.gaussian_filter_2d(sigma, per_channel=True)
    chunk.array[...] = dev.tensor.cpu().numpy()
    return chunk
