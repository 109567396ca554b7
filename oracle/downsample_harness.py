"""Run the REAL vendored downsampler of the reference (reference lib/igneous/downsample.py; TEST INFRASTRUCTURE, needs the
reference tree).

Two shims, nothing else changed:
* ``np.cast`` is gone from numpy 2; the module sees a numpy whose ``cast[dt](x)`` is ``np.asarray(x).astype(dt)``.
* :func:`segmentation` with ``floor_division=True`` runs a copy of the module's source in which the two ``factor / 2`` of
  the recursion read ``factor // 2``: the reference's ``factor / 2`` is a float, on which ``x & (x - 1)`` raises a TypeError
  as soon as a second level is reached.  The unmodified module records which factors raise.

:func:`thumbnail` drives the reference's own ``downsample_and_upload`` (lib/igneous/tasks.py) as
``save-precomputed --create-thumbnail`` calls it (save_precomputed.py:104-139), with a small recording stand-in for the
CloudVolume object and numpy stand-ins for the two ``cloudvolume.lib`` helpers it imports (``min2``, ``Vec``).

The module takes the arrays its callers give it: 3-D ones for 3-D factors, and for planar factors (one axis 1) the channel-last
``a[..., None]`` with the factor ``(fz, fy, fx, 1)`` -- its 2x2 path indexes a fourth axis and its 3-D path asserts that every
axis, the channel one included, is even.
"""
import os
import sys
import types

import numpy as np

from oracle import reference_harness as H

available = H.available
SOURCE = os.path.join(H.REFERENCE_ROOT, "chunkflow", "lib", "igneous", "downsample.py")
_modules = {}


def _numpy_with_cast():
    shim = types.ModuleType("numpy_with_cast")
    shim.__dict__["__getattr__"] = lambda name: getattr(np, name)

    class Cast:
        def __getitem__(self, dtype):
            return lambda x: np.asarray(x).astype(dtype)

    shim.cast = Cast()
    return shim


def module(floor_division=False):
    """The vendored module, loaded from the reference tree (with ``factor // 2`` when ``floor_division``)."""
    if floor_division not in _modules:
        if not available():
            raise RuntimeError(f"reference tree not found at {H.REFERENCE_ROOT}")
        with open(SOURCE) as f:
            text = f.read()
        if floor_division:
            assert text.count("factor / 2") == 2, "the recursion of the vendored module changed"
            text = text.replace("factor / 2", "factor // 2")
        m = types.ModuleType("reference_igneous_downsample" + ("_floor" if floor_division else ""))
        m.__file__ = SOURCE
        exec(compile(text, SOURCE, "exec"), m.__dict__)
        m.np = _numpy_with_cast()
        _modules[floor_division] = m
    return _modules[floor_division]


def average(a, factor):
    """downsample_with_averaging of the (z, y, x) array."""
    return np.asarray(module().downsample_with_averaging(np.array(a, copy=True), tuple(int(v) for v in factor)))


def segmentation(a, factor, floor_division=False):
    """downsample_segmentation of the (z, y, x) array in the form its callers use -> (z, y, x) result; exceptions pass."""
    f = tuple(int(v) for v in factor)
    m = module(floor_division)
    a = np.array(a, copy=True)
    out = np.asarray(m.downsample_segmentation(a[..., None], f + (1,)) if 1 in f else m.downsample_segmentation(a, f))
    return out[..., 0] if out.ndim == 4 else out   # a later 2x2 level of a 3-D factor grows the channel axis too


def raises(a, factor, floor_division=False):
    """The name of the exception the module raises for this input, or '' when it does not."""
    try:
        segmentation(a, factor, floor_division)
    except Exception as exc:   # noqa: BLE001 -- recorded, not handled
        return type(exc).__name__
    return ""


class RecordingVolume:
    """What downsample_and_upload reads of a CloudVolume (an image layer, mips 0..11 with 4^3 underlying chunks, a large
    volume) and every write it makes, as (mip, slices, array)."""
    layer_type = "image"
    volume_size = np.array([1 << 20] * 3)
    available_mips = range(0, 12)

    def __init__(self):
        self.mip = 0
        self.writes = []

    def mip_underlying(self, mip):
        return np.array([4, 4, 4])

    def __setitem__(self, slices, image):
        self.writes.append((self.mip, slices, np.array(image)))


def thumbnail(affinity, max_mip=6):
    """The thumbnail of a (c, z, y, x) float32 affinity map as save_precomputed.py:104-139 makes it (last channel, times 255,
    uint8, transposed to x, y, z; axis 'z', skip_first, only_last_mip) -> (mip of the level written, (z, y, x) uint8 array)."""
    if not available():
        raise RuntimeError(f"reference tree not found at {H.REFERENCE_ROOT}")
    H.import_reference()
    lib = sys.modules["cloudvolume.lib"]
    saved = {k: getattr(lib, k) for k in ("min2", "Vec") if hasattr(lib, k)}
    lib.min2 = lambda a, b: np.minimum(np.asarray(a), np.asarray(b))
    lib.Vec = lambda *a: np.array(a)
    try:
        import chunkflow.lib.igneous.downsample as ref_downsample
        from chunkflow.lib.igneous import tasks
        from chunkflow.lib.cartesian_coordinate import BoundingBox, Cartesian
    finally:
        for k in ("min2", "Vec"):
            if k in saved:
                setattr(lib, k, saved[k])
            else:
                delattr(lib, k)
    ref_downsample.np = module().np
    image = np.asarray(affinity)[-1]
    image = np.transpose((image * 255).astype(np.uint8))
    vol = RecordingVolume()
    bounds = BoundingBox.from_delta(Cartesian(0, 0, 0), Cartesian(*image.shape))
    tasks.downsample_and_upload(image, bounds, vol, np.array(image.shape), mip=0, max_mip=max_mip, axis='z', skip_first=True,
                                only_last_mip=True)
    assert len(vol.writes) == 1, "only the last mip is written"
    mip, _, out = vol.writes[0]
    return mip, np.transpose(out)
