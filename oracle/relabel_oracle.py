"""Numpy restatement of the reference's segmentation clean-up (TEST INFRASTRUCTURE; DESIGN.md section 0, row f6).

The reference's own code (chunk/segmentation.py) is pinned by golden vectors recorded from it
(tests/golden/relabel_reference.npz, oracle/relabel_harness.py).  The four ``fastremap`` functions it calls belong to a
third-party package that is not part of the reference tree; they are restated here from their published behaviour and are
flagged PARITY UNPINNED: nothing in this repository has been compared with the real package.

Ids are compared as the uint64 values ``astype(np.uint64)`` gives (the convention of oracle/evaluation_oracle.py).
"""
import json

import numpy as np


def _u64(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a).astype(np.uint64, copy=False))


def _ids_u64(ids) -> np.ndarray:
    return np.array([int(i) % 2 ** 64 for i in ids], dtype=np.uint64)


# ---- fastremap, restated (PARITY UNPINNED) ------------------------------------------------------------------------
def unique(array, return_counts=False, return_index=False):
    """fastremap.unique(a, return_counts=True): ids ascending (as unsigned), their voxel counts; ``return_index`` adds the
    C-order linear index of each id's first voxel (what the device table holds besides the count).  PARITY UNPINNED."""
    a = np.asarray(array)
    ids, first, counts = np.unique(_u64(a).ravel(), return_index=True, return_counts=True)
    out = [ids.astype(a.dtype)]
    if return_index:
        out.append(first)
    if return_counts:
        out.append(counts)
    return out[0] if len(out) == 1 else tuple(out)


def mask(array, ids):
    """fastremap.mask(a, ids): the listed ids become 0, dtype unchanged.  PARITY UNPINNED."""
    a = np.asarray(array)
    out = a.copy()
    out[np.isin(_u64(a), _ids_u64(ids))] = 0
    return out


def mask_except_ids(array, ids):
    """fastremap.mask_except(a, ids): every id not listed becomes 0, dtype unchanged.  PARITY UNPINNED."""
    a = np.asarray(array)
    out = a.copy()
    out[~np.isin(_u64(a), _ids_u64(ids))] = 0
    return out


def renumber(array, preserve_zero=True):
    """fastremap.renumber(a, preserve_zero=True): non-zero ids become 1..N in the order in which they are first met in a
    C-order raster scan, 0 stays 0.  Returns (renumbered uint64 array, N).  PARITY UNPINNED."""
    assert preserve_zero
    a = _u64(array)
    ids, first, inverse = np.unique(a.ravel(), return_index=True, return_inverse=True)
    nz = ids != 0
    order = np.argsort(first[nz], kind="stable")        # survivors by first voxel
    new = np.zeros(ids.size, np.uint64)
    new_nz = np.empty(int(nz.sum()), np.uint64)
    new_nz[order] = np.arange(1, order.size + 1, dtype=np.uint64)
    new[nz] = new_nz
    return new[inverse].reshape(a.shape), int(order.size)


# ---- the reference's Segmentation methods -------------------------------------------------------------------------
def mask_fragments(array, voxel_num_threshold):
    """Segmentation.mask_fragments (reference chunk/segmentation.py:86-90): ids with ``count <= threshold`` become 0 (`<=`, not
    the CLI help's "less than"; 0 is an ordinary entry of both printed numbers).  -> (array, printed line)."""
    uniq, counts = unique(array, return_counts=True)
    fragment_ids = uniq[counts <= voxel_num_threshold]                                                   # :88
    line = (f'masking out {len(fragment_ids)} fragments in {len(uniq)} with a percentage of '
            f'{len(fragment_ids) / len(uniq)}\n')                                                         # :89
    return mask(array, fragment_ids), line                                                               # :90


def parse_selected_obj_ids(selected_obj_ids):
    """The id selection of Segmentation.mask_except (reference chunk/segmentation.py:93-107) -> (list of ints or None,
    printed text).  A ``.json`` path is read as a local file (the reference goes through CloudFiles)."""
    if selected_obj_ids is None:
        return None, 'we have not selected any objects to mask out.\n'                                   # :93-95
    if isinstance(selected_obj_ids, str) and selected_obj_ids.endswith('.json'):                         # :97-103
        with open(selected_obj_ids) as f:
            ids = set(json.load(f))
        assert len(ids) > 0
        return sorted(ids), f'number of selected objects: {len(ids)}\n'
    if isinstance(selected_obj_ids, str):                                                                # :104-107
        return sorted(set(int(i) for i in selected_obj_ids.split(','))), ''
    return list(selected_obj_ids), ''


def mask_except(array, selected_obj_ids):
    """Segmentation.mask_except (reference chunk/segmentation.py:92-109) -> (array, printed text)."""
    ids, text = parse_selected_obj_ids(selected_obj_ids)
    if ids is None:
        return np.asarray(array), text
    return mask_except_ids(array, ids), text                                                             # :109


def remap(array, base_id=0):
    """Segmentation.remap (reference chunk/segmentation.py:69-84): renumber, astype(uint64), add ``base_id`` to the non-zero
    voxels when it is > 0, return the maximum of the result (0 for an all-zero chunk whatever ``base_id``: the reference's
    value).  -> (uint64 array, new_base_id)."""
    out, _ = renumber(array)                                                                             # :78-80
    if base_id > 0:
        out[out > 0] += np.uint64(base_id)                                                               # :81-82
    return out, int(out.max())                                                                           # :83-84


def mask_out_objects(array, dust_size_threshold=None, selected_obj_ids=None):
    """The body of `mask-out-objects` (reference flow/flow.py:2044-2047): dust first, then the keep-list.
    -> (array, printed text)."""
    text = ''
    if dust_size_threshold is not None:
        array, line = mask_fragments(array, dust_size_threshold)
        text += line
    if selected_obj_ids is not None:
        array, line = mask_except(array, selected_obj_ids)
        text += line
    return array, text
