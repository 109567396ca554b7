"""CPU restatement of `fill-segmentation-holes` (reference chunkflow/plugins/fill_segmentation_holes.py, which returns
``fill_voids.fill(seg.array)`` with the chunk's properties).  fill_voids is NOT vendored in the reference tree and not installed
here, so its 0/1 output is restated from its published behaviour, not pinned.  The hole mask is pinned: it equals live
``scipy.ndimage.binary_fill_holes(arr != 0)``, whose default structure is the 6-connected cross.

Rules.  Every connectivity is 6 (face neighbours).  "Outside" is the space beyond the chunk's six faces: a voxel on a face
reaches it.

* ``binary`` (the reference plugin): foreground is every voxel ``!= 0`` (float32: -0.0 is background, NaN foreground).  A
  background voxel is a hole when no 6-connected path of background voxels leads from it to outside.  The result has the
  input's dtype: 1 for foreground and holes, 0 elsewhere.  Count: the holes.
* Per-object modes (an extension: what kimimaro's and fastmorph's ``fill_holes`` are for).  An object is a 6-connected
  component of one non-zero id.  Object O encloses voxel v (v not in O) when every 6-connected path from v to outside passes
  through O, i.e. v lies in ``binary_fill_holes(O) & ~O``.  The objects that enclose a voxel are nested (if O2 lies inside O1,
  ``binary_fill_holes(O2)`` is strictly inside ``binary_fill_holes(O1)``), so they are ordered here by the size of their
  filled mask: the innermost has the smallest.
  - ``keep-enclosed``: every voxel with id 0 enclosed by at least one object takes the id of the innermost one; non-zero
    voxels do not change.  Count: the enclosed zeros.
  - ``remove-enclosed``: every enclosed voxel, whatever its id, takes the id of the outermost encloser.  Count: every enclosed
    voxel.

Brute force on purpose (``ndimage.label`` per id, ``binary_fill_holes`` per component): it shares nothing with the native
algorithm (component graph, articulation points), so that the two derivations check each other.  Small volumes only.
"""
import numpy as np
from scipy import ndimage

MODES = ("binary", "keep-enclosed", "remove-enclosed")
BINARY_DTYPES = (np.bool_, np.uint8, np.int32, np.uint32, np.int64, np.uint64, np.float32)
OBJECT_DTYPES = (np.uint32, np.int32, np.uint64, np.int64)


def check(arr: np.ndarray, mode: str) -> None:
    if mode not in MODES:
        raise ValueError(f"fill holes: the mode is one of {MODES}, not {mode!r}")
    dtypes = BINARY_DTYPES if mode == "binary" else OBJECT_DTYPES
    if arr.dtype not in [np.dtype(d) for d in dtypes]:
        raise TypeError(f"fill holes: {mode} mode takes {', '.join(np.dtype(d).name for d in dtypes)} voxels, not {arr.dtype}")
    if arr.ndim != 3:
        raise ValueError(f"fill holes: a (z, y, x) chunk, not {arr.ndim}-D")


def holes(arr: np.ndarray) -> np.ndarray:
    """The binary rule's hole mask."""
    fg = np.asarray(arr) != 0
    return ndimage.binary_fill_holes(fg) & ~fg


def objects(arr: np.ndarray):
    """Every object as (id, filled size, enclosed mask): ``binary_fill_holes(O) & ~O`` over the whole chunk.  The fill is
    computed on the object's bounding box, which gives the same mask: every voxel outside the box reaches outside without
    crossing O, and so does every voxel on the box's border that is not in O."""
    arr = np.asarray(arr)
    out = []
    for v in np.unique(arr):
        if v == 0:
            continue
        lab, k = ndimage.label(arr == v)   # default structure: the 6-connected cross
        for sl, j in zip(ndimage.find_objects(lab), range(1, k + 1)):
            o = lab[sl] == j
            filled = ndimage.binary_fill_holes(o)
            enclosed = np.zeros(arr.shape, bool)
            enclosed[sl] = filled & ~o
            out.append((v, int(filled.sum()), enclosed))
    return out


def enclosers(arr: np.ndarray, index) -> list:
    """(id, filled size) of every object that encloses the voxel at ``index``, innermost first."""
    return sorted(((v, s) for v, s, e in objects(arr) if e[index]), key=lambda t: t[1])


def fill(arr: np.ndarray, mode: str = "binary"):
    """-> (filled chunk in the input's dtype, number of voxels the rule assigns)."""
    arr = np.asarray(arr)
    check(arr, mode)
    if mode == "binary":
        h = holes(arr)
        return ((arr != 0) | h).astype(arr.dtype), int(h.sum())
    out = arr.copy()
    assigned = np.zeros(arr.shape, bool)
    # keep-enclosed: largest filled mask first, so that the innermost encloser writes last; remove-enclosed: smallest first
    for v, _, e in sorted(objects(arr), key=lambda t: t[1], reverse=(mode == "keep-enclosed")):
        if mode == "keep-enclosed":
            e = e & (arr == 0)
        out[e] = v
        assigned |= e
    return out, int(assigned.sum())
