"""Run the REAL reference plugin ``plugins/clahe.py`` (TEST INFRASTRUCTURE, needs the reference tree and OpenCV): the file is
loaded from the reference tree as its plugin operator loads it, and ``execute`` equalizes every z section of a reference
``Chunk`` in place with the module's ``clahe`` object.  Other parameters run through the plugin's own loop by replacing that
object with ``cv2.createCLAHE(clip_limit, tile_grid_size)``.
"""
import contextlib
import io
import os
import types

import numpy as np

from oracle import reference_harness as H

_module = None


def available() -> bool:
    try:
        import cv2  # noqa: F401
    except ImportError:
        return False
    return H.available()


def _plugin():
    global _module
    if _module is None:
        H.import_reference()
        path = os.path.join(H.REFERENCE_ROOT, "chunkflow", "plugins", "clahe.py")
        m = types.ModuleType("reference_plugin_clahe")
        m.__file__ = path
        with open(path) as f:
            exec(compile(f.read(), path, "exec"), m.__dict__)
        _module = m
    return _module


def plugin_defaults():
    """(clipLimit, tileGridSize) of the reference module."""
    m = _plugin()
    return float(m.clipLimit), tuple(m.tileGridSize)


def clahe_plugin(array, clip_limit=None, tile_grid_size=None):
    """plugins/clahe.execute(Chunk(array)) -> the chunk's array; the module's own clahe object where both are None."""
    import cv2
    Chunk = H.import_reference()[1]
    m = _plugin()
    default = m.clahe
    if clip_limit is not None or tile_grid_size is not None:
        m.clahe = cv2.createCLAHE(clipLimit=m.clipLimit if clip_limit is None else clip_limit,
                                  tileGridSize=m.tileGridSize if tile_grid_size is None else tuple(tile_grid_size))
    try:
        chunk = Chunk(np.array(array, copy=True))
        with contextlib.redirect_stderr(io.StringIO()):
            out = m.execute(chunk)
        assert out is chunk
        return np.asarray(out.array)
    finally:
        m.clahe = default
