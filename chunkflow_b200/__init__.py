"""chunkflow_b200 -- H100-native implementation of chunkflow's ``inference`` hot path.

Host side in Python (mirrors the reference's operator / plugin interface), hot path as
hand-written sm_90a CUDA kernels behind a C-ABI shared library
(``include/chunkflow_b200.h``, loaded with ctypes by :mod:`chunkflow_b200._native`).
"""
from .chunk import Chunk  # noqa: F401
from .lib.cartesian_coordinate import Cartesian, to_cartesian  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    if name == "Inferencer":
        from .flow.divid_conquer.inferencer import Inferencer
        return Inferencer
    if name == "DeviceChunk":
        from .chunk.device import DeviceChunk
        return DeviceChunk
    raise AttributeError(name)
