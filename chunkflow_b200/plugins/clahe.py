"""Contrast-limited adaptive histogram equalization of every section -- drop-in for the reference's plugin
``chunkflow/plugins/clahe.py``, which runs ``cv2.createCLAHE(clipLimit=20.0, tileGridSize=(512, 512)).apply`` on every z.

Same module constants, same signature, same return value: the chunk itself, its array rewritten in place, bit-identical to
OpenCV.  The sections are equalized by CUDA kernels (``csrc/clahe_kernels.cuh``); a host ``Chunk`` goes to the GPU and back,
a ``DeviceChunk`` has the result copied into its tensor.  There is no CPU fallback.
"""
from chunkflow_b200.chunk import Chunk

clipLimit = 20.0
tileGridSize = (512, 512)


def execute(img: Chunk):
    from chunkflow_b200.chunk.device import DeviceChunk
    assert img.is_image
    if isinstance(img, DeviceChunk):
        img.tensor.copy_(img.clahe(clipLimit, tileGridSize).tensor)
        return img
    out = DeviceChunk.from_chunk(img).clahe(clipLimit, tileGridSize)
    img.array[...] = out.tensor.cpu().numpy()
    return img
