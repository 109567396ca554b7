"""Agglomeration including the watershed step -- drop-in for the reference's plugin
``chunkflow/plugins/agglomerate.py`` (``execute``, lines 8-48), which calls ``waterz.agglomerate``.

Same signature, same return value (a list with one segmentation ``Chunk``, uint64 like waterz's).  The affinity map is moved to
the GPU; watershed, region-graph statistics and the final relabel are CUDA kernels (``csrc/watershed_kernels.cuh``), the merge
loop over the fragment graph runs in the native library on the host like waterz's C++.  There is no CPU fallback.  Two of
waterz's scoring functions are implemented: the mean affinity the reference's plugin defaults to, and the histogram-quantile
family ``OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B[, I]>>`` (lsd's ``hist_quant_50`` and
``hist_quant_50_initmax``); any other raises NotImplementedError.  waterz is not vendored in the reference tree: parity is
against its published algorithm as restated in ``oracle/agglomeration_oracle.py`` and
``oracle/agglomeration_quantile_oracle.py`` ("parity unpinned"; deviations listed there).
"""
import numpy as np

from chunkflow_b200.chunk import Chunk

SCORING_FUNCTION = 'OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>'


def execute(affs: Chunk,
            fragments: np.ndarray = None,
            threshold: float = 0.7,
            aff_threshold_low: float = 0.001,
            aff_threshold_high: float = 0.9999,
            scoring_function: str = SCORING_FUNCTION,
            flip_channel: bool = True,
            device="cuda:0"):
    """
    Parameters:
    -----------
    affs: affinity map with 4 dimensions: channel, z, y, x (chunkflow's channel order is x, y, z: ``flip_channel``)
    fragments: optional (z, y, x) integer array of supervoxels to start from instead of the watershed
    """
    from chunkflow_b200.chunk.device import DeviceChunk, parse_scoring_function
    parse_scoring_function(scoring_function)   # refused before anything moves to the GPU
    import torch
    arr = np.ascontiguousarray(np.asarray(affs.array if isinstance(affs, Chunk) else affs), dtype=np.float32)  # reference :33
    assert arr.ndim == 4 and arr.shape[0] == 3, 'affinity map with 4 dimensions: channel (3), z, y, x'
    dev = DeviceChunk(torch.from_numpy(arr).to(device), voxel_offset=getattr(affs, 'voxel_offset', None),
                      voxel_size=getattr(affs, 'voxel_size', None), layer_type='affinity_map')
    frag = None
    if fragments is not None:
        f = np.asarray(fragments.array if isinstance(fragments, Chunk) else fragments)
        assert f.shape == arr.shape[1:] and np.issubdtype(f.dtype, np.integer), 'fragments: (z, y, x) integer array'
        if f.size and (int(f.max()) >= 2 ** 31 or int(f.min()) < 0):
            raise ValueError('fragment ids must be in [0, 2^31) on the device')
        frag = DeviceChunk(torch.from_numpy(np.ascontiguousarray(f.astype(np.int32))).to(device), layer_type='segmentation')
        frag.num_components = int(f.max()) if f.size else 0
    seg = dev.agglomerate(threshold=threshold, aff_threshold_low=aff_threshold_low, aff_threshold_high=aff_threshold_high,
                          fragments=frag, flip_channel=flip_channel, scoring_function=scoring_function)
    out = seg.tensor.cpu().numpy().view(np.uint32).astype(np.uint64)   # waterz returns uint64
    vo = getattr(affs, 'voxel_offset', None)
    return [Chunk(out, voxel_offset=vo, voxel_size=getattr(affs, 'voxel_size', None))]
