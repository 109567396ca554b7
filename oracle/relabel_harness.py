"""Run the REAL reference ``Segmentation.mask_fragments / mask_except / remap`` (TEST INFRASTRUCTURE; needs the reference tree).

``chunk/segmentation.py`` calls four functions of ``fastremap``, a third-party package that is neither in the reference tree
nor installed here.  oracle/evaluation_harness.py registers an empty ``fastremap`` module so that the file imports; this
harness fills it with numpy stand-ins of the package's published behaviour (PARITY UNPINNED, like oracle/relabel_oracle.py),
so that everything AROUND those calls is the reference's own code: the ``<=`` of the dust test, the printed line, the parsing
of the id string, ``astype(np.uint64)``, the base-id addition and the returned maximum.
"""
import io
import sys
from contextlib import redirect_stdout

import numpy as np

from oracle import evaluation_harness as EH

available = EH.available


def _u64(a):
    return np.asarray(a).astype(np.uint64, copy=False)


def _ids(ids):
    return np.array([int(i) % 2 ** 64 for i in ids], dtype=np.uint64)


def _unique(a, return_counts=False):
    ids, counts = np.unique(_u64(a), return_counts=True)
    ids = ids.astype(np.asarray(a).dtype)
    return (ids, counts) if return_counts else ids


def _mask(a, ids):
    out = np.array(a, copy=True)
    out[np.isin(_u64(a), _ids(ids))] = 0
    return out


def _mask_except(a, ids):
    out = np.array(a, copy=True)
    out[~np.isin(_u64(a), _ids(ids))] = 0
    return out


def _renumber(a, preserve_zero=True, in_place=False):
    assert preserve_zero
    flat = _u64(a).ravel()
    ids, first, inverse = np.unique(flat, return_index=True, return_inverse=True)
    by_first = np.argsort(first, kind="stable")
    new = np.zeros(ids.size, np.uint64)
    k = 0
    for j in by_first:
        if ids[j] != 0:
            k += 1
            new[j] = k
    out = new[inverse].reshape(np.shape(a)).astype(np.asarray(a).dtype)
    mapping = {int(i): int(n) for i, n in zip(ids, new)}
    if in_place:
        a[...] = out
        return a, mapping
    return out, mapping


def import_reference_segmentation():
    """Returns (Segmentation, Chunk) of the real reference with the fastremap stand-ins in place."""
    Segmentation, Chunk, _ = EH.import_reference_evaluation()
    fr = sys.modules["fastremap"]
    fr.unique, fr.mask, fr.mask_except, fr.renumber = _unique, _mask, _mask_except, _renumber
    return Segmentation, Chunk


def run(method: str, array, *args):
    """Call one reference method on a copy of ``array`` -> (resulting array, returned value, printed text)."""
    Segmentation, Chunk = import_reference_segmentation()
    seg = Segmentation(np.array(array, copy=True))
    buf = io.StringIO()
    with redirect_stdout(buf):
        ret = getattr(seg, method)(*args)
    return seg.array, ret, buf.getvalue()
