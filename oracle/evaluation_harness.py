"""Import the REAL reference `Segmentation` and gala's evaluate module (TEST INFRASTRUCTURE; needs the reference tree).

On top of oracle/reference_harness.py's stubs: ``chunk/segmentation.py`` imports fastremap and cloudfiles (unused by
``evaluate``), and gala's evaluate.py imports ``skimage.segmentation.relabel_sequential``, which ``raw_edit_distance`` calls
(evaluate.py:200-201).  skimage is not installed offline, so a small numpy implementation of its documented behaviour
stands in: non-zero labels renumbered 1..N in increasing order, 0 stays 0.
"""
import sys
import types

import numpy as np

from oracle import reference_harness as H

available = H.available


def relabel_sequential(label_field, offset=1):
    a = np.asarray(label_field)
    uniq = np.unique(a)
    nz = uniq[uniq != 0]
    out = np.zeros(a.shape, np.int64)
    m = a != 0
    out[m] = np.searchsorted(nz, a[m]) + offset
    fw = inv = None   # the reference uses only the relabelled array
    return out, fw, inv


def import_reference_evaluation():
    """Returns (Segmentation, Chunk, gala evaluate module) of the real reference."""
    def stub(name, **attrs):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            sys.modules[name] = m
        return sys.modules[name]

    H.import_reference()   # stubs h5py, cloudvolume, skimage, ... and puts the reference tree on sys.path
    stub("fastremap")
    stub("cloudfiles", CloudFiles=type("CloudFiles", (), {}))
    sk = sys.modules["skimage"]
    sk.segmentation = stub("skimage.segmentation", relabel_sequential=relabel_sequential)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from chunkflow.chunk import Chunk
        from chunkflow.chunk.segmentation import Segmentation
        from chunkflow.lib.gala import evaluate
    return Segmentation, Chunk, evaluate
