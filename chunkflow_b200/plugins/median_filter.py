"""Median filter -- drop-in for the reference's plugin ``chunkflow/plugins/median_filter.py`` (``execute``, lines 4-7),
which returns ``[scipy.ndimage.median_filter(chunk, size=size, mode=mode)]``.

Same signature, same return value: a list with the filtered array (the reference's plugin operator turns it back into a
chunk with the input's offset and voxel size), bit-identical to scipy.  The filter runs as CUDA kernels
(``csrc/filter_kernels.cuh``); a host chunk or array goes to the GPU and back, a ``DeviceChunk`` gives a ``DeviceChunk``.
There is no CPU fallback.
"""
import numpy as np


def execute(chunk, size: tuple = (3, 1, 1), mode: str = 'reflect'):
    import torch
    from chunkflow_b200.chunk.device import DeviceChunk
    print('median filtering of chunk...')
    if isinstance(chunk, DeviceChunk):
        return [chunk.median_filter(size=size, mode=mode)]
    arr = np.ascontiguousarray(np.asarray(chunk))
    out = DeviceChunk(torch.from_numpy(arr).to("cuda:0")).median_filter(size=size, mode=mode)
    return [out.tensor.cpu().numpy()]
