"""TEASAR skeletons of a segmentation chunk -- drop-in for the reference's plugin ``chunkflow/plugins/skeletonize.py``, which runs
``kimimaro.skeletonize`` and writes every skeleton's precomputed bytes as ``{id}:{bbox}`` through CloudFiles.

Same signature and return value (``{id: skeleton}``, here ``chunkflow_b200.flow.skeleton.Skeleton``).  The skeletons follow the
rules of ``oracle/skeleton_oracle.py`` on the GPU (``csrc/skeleton.cu``): they are not kimimaro's, and the reference's handling
of zyx / xyz order is not imitated (``voxel_size`` is z, y, x and the vertices are x, y, z).  A host ``Chunk`` goes to the GPU
for the call.  ``output_path`` is a local directory or ``file://`` URL; the fragments' vertices are shifted by voxel offset *
voxel size into the volume's frame.  There is no CPU fallback.
"""
from chunkflow_b200.chunk import Chunk


def skeletonize(seg: Chunk, voxel_size):
    from chunkflow_b200.chunk.device import DeviceChunk
    dev = seg if isinstance(seg, DeviceChunk) else DeviceChunk.from_chunk(seg)
    return dev.skeletonize(voxel_size=voxel_size)


def execute(seg: Chunk, voxel_size: tuple, output_path: str = None):
    """Create skeleton fragments from segmentation."""
    from chunkflow_b200.flow.skeleton import write_fragments
    if seg is None:
        print('no segmentation, skip computation.')
        return None
    print('skeletonize segmentation...')
    skels = skeletonize(seg, voxel_size)
    if output_path is not None:
        write_fragments(skels, output_path, tuple(seg.voxel_offset), seg.shape[-3:], voxel_size)
    return skels
