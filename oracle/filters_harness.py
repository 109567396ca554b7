"""Run the REAL reference code of the two smoothing operators (TEST INFRASTRUCTURE, needs the reference tree):
``Chunk.gaussian_filter_2d`` (chunk/base.py:846-853, what the `gaussian-filter` command calls), and the plugin files
``plugins/gaussian_filter.py`` and ``plugins/median_filter.py``, loaded from the reference tree as its plugin operator loads
them.  All three call scipy.ndimage, which is installed here.
"""
import contextlib
import io
import os
import types

import numpy as np

from oracle import reference_harness as H

available = H.available
_plugins = {}


def _plugin(name):
    if name not in _plugins:
        H.import_reference()
        path = os.path.join(H.REFERENCE_ROOT, "chunkflow", "plugins", f"{name}.py")
        m = types.ModuleType(f"reference_plugin_{name}")
        m.__file__ = path
        with open(path) as f:
            exec(compile(f.read(), path, "exec"), m.__dict__)
        _plugins[name] = m
    return _plugins[name]


def gaussian_filter_2d(array, sigma):
    """The reference's Chunk(array).gaussian_filter_2d(sigma) -> the filtered array (the method works in place)."""
    Chunk = H.import_reference()[1]
    chunk = Chunk(np.array(array, copy=True))
    chunk.gaussian_filter_2d(sigma)
    return np.asarray(chunk.array)


def gaussian_plugin(array, sigma=1.0):
    """plugins/gaussian_filter.execute(Chunk(array), sigma) -> the returned chunk's array; the input is checked unchanged."""
    Chunk = H.import_reference()[1]
    chunk = Chunk(np.array(array, copy=True))
    out = _plugin("gaussian_filter").execute(chunk, sigma=sigma)
    assert np.array_equal(chunk.array, array), "the plugin changed its input without inplace"
    return np.asarray(out.array)


def median_plugin(array, size=(3, 1, 1), mode="reflect"):
    """plugins/median_filter.execute(Chunk(array), size, mode) -> its one output array."""
    Chunk = H.import_reference()[1]
    with contextlib.redirect_stdout(io.StringIO()):
        out = _plugin("median_filter").execute(Chunk(np.array(array, copy=True)), size=size, mode=mode)
    assert isinstance(out, list) and len(out) == 1
    return np.asarray(out[0])
