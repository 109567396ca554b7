"""numpy restatement of `evaluate-segmentation` (DESIGN.md section 0, row f5): Segmentation.evaluate(groundtruth, size_threshold)
(reference chunk/segmentation.py:33-67) -> the vendored gala metrics (reference lib/gala/evaluate.py).  Written from the
formulas, not from the reference's code; pinned to the real reference by tests/golden/evaluate_reference.npz
(tests/golden/make_golden_evaluate.py) and, where the reference tree exists, by tests/test_evaluate_oracle.py.

With c the counts of the sparse contingency table of (seg id, gt id) pairs (contingency_table, evaluate.py:212-249):

* rand index, adjusted rand index, Fowlkes-Mallows index: the table with NOTHING ignored (0 is an ordinary label);
  rand_values (:1183-1223) gives a = (S1 - n) / 2.0, b = (S2 - S1) / 2, c = (S3 - S1) / 2, d = (S1 + n**2 - S2 - S3) / 2
  with S1 = sum c^2, S2 / S3 the sums of the squared row / column sums; then the formulas at :1248, :1274-1275, :1300 in
  gala's operation order.
* variation of information (vi -> split_vi -> vi_tables, :623-691, :1049-1101): ignore_x = ignore_y = [0] drops every voxel
  with a 0 on EITHER side; over the N' remaining voxels, with xl(v) = sum v log2 v:
  VI = ((xl(r') - xl(c)) + (xl(s') - xl(c))) / N'.
* edit distance (raw_edit_distance, :183-209): (K - N_seg, 0.0), K = pairs with both ids != 0 and count > size_threshold,
  N_seg = distinct non-zero seg ids.  The second element is always 0.0 (the reference slices the rows of a 1 x N matrix).

0/0 gives NaN (numpy's float division), as in the reference.  Everything is computed from uint64 ids (astype(np.uint64)), so
ids of any size work -- the reference itself fails on ids of about 2^40 and more.
"""
from __future__ import annotations

import numpy as np


def as_labels(a) -> np.ndarray:
    """What the reference does first (segmentation.py:39-45): astype(np.uint64), flattened."""
    return np.ascontiguousarray(np.asarray(a).astype(np.uint64)).ravel()


def contingency_triples(seg, gt):
    """(seg ids, gt ids, counts) of the contingency table, sorted by (seg, gt); the counts are uint64."""
    s, g = as_labels(seg), as_labels(gt)
    if s.shape != g.shape:
        raise ValueError("segmentation and ground truth must have the same shape")
    if s.size == 0:
        e = np.zeros(0, np.uint64)
        return e, e.copy(), e.copy()
    su, si = np.unique(s, return_inverse=True)
    gu, gi = np.unique(g, return_inverse=True)
    # dense (seg rank, gt rank) key: its order is the (seg, gt) order; su.size * gu.size <= n^2 < 2^64
    key, counts = np.unique(si.ravel().astype(np.uint64) * np.uint64(gu.size) + gi.ravel().astype(np.uint64), return_counts=True)
    return su[key // np.uint64(gu.size)], gu[key % np.uint64(gu.size)], counts.astype(np.uint64)


def _xlog2(v: np.ndarray) -> float:
    v = np.sort(v[v > 1]).astype(np.float64)   # summed in value order: the same result under any relabelling
    return float(np.sum(v * np.log2(v)))


def statistics(seg_ids, gt_ids, counts, size_threshold=1000) -> dict:
    """The exact integer statistics and the three entropy sums the scores need, from the table's triples."""
    seg_ids, gt_ids = np.asarray(seg_ids, np.uint64), np.asarray(gt_ids, np.uint64)
    c = np.asarray(counts, np.uint64)
    both = (seg_ids != 0) & (gt_ids != 0)
    _, rinv = np.unique(seg_ids, return_inverse=True)
    _, cinv = np.unique(gt_ids, return_inverse=True)
    c_both = np.where(both, c, np.uint64(0)).astype(np.uint64)
    rows, cols = _sum_by(rinv, c), _sum_by(cinv, c)                 # marginals over all voxels
    rows_nz, cols_nz = _sum_by(rinv, c_both), _sum_by(cinv, c_both)  # r', s': over the voxels with both ids != 0
    py = lambda a: sum(int(v) * int(v) for v in a)   # exact: n < 2^32 keeps every sum below 2^64
    thr = float(size_threshold)
    return dict(
        n=int(sum(int(v) for v in c)),
        sum_sq_pairs=py(c), sum_sq_rows=py(rows), sum_sq_cols=py(cols),
        n_both_nonzero=int(sum(int(v) for v in c[both])),
        seg_ids=int(np.count_nonzero(np.unique(seg_ids) != 0)),
        gt_ids=int(np.count_nonzero(np.unique(gt_ids) != 0)),
        pairs=int(c.size),
        pairs_over_threshold=int(np.count_nonzero(both & ~(c.astype(np.float64) <= thr))),
        xlog_pairs=_xlog2(c[both]), xlog_rows=_xlog2(rows_nz), xlog_cols=_xlog2(cols_nz),
    )


def _sum_by(inverse, values):
    out = np.zeros(int(inverse.max()) + 1 if inverse.size else 0, np.uint64)
    np.add.at(out, inverse.ravel(), np.asarray(values, np.uint64))
    return out


def scores(st: dict) -> dict:
    """The five scores from the statistics, in gala's operation order (float64 throughout)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        n = np.float64(st["n"])
        sum1, sum2, sum3 = np.float64(st["sum_sq_pairs"]), np.float64(st["sum_sq_rows"]), np.float64(st["sum_sq_cols"])
        a = (sum1 - n) / 2.0
        b = (sum2 - sum1) / 2
        c = (sum3 - sum1) / 2
        d = (sum1 + n ** 2 - sum2 - sum3) / 2
        ri = (a + d) / (a + b + c + d)
        nk = a + b + c + d
        ari = (nk * (a + d) - ((a + b) * (a + c) + (c + d) * (b + d))) / (nk ** 2 - ((a + b) * (a + c) + (c + d) * (b + d)))
        fm = a / (np.sqrt((a + b) * (a + c)))
        xc, xr, xs = np.float64(st["xlog_pairs"]), np.float64(st["xlog_rows"]), np.float64(st["xlog_cols"])
        vi = ((xr - xc) + (xs - xc)) / np.float64(st["n_both_nonzero"])
    edit = (np.float64(st["pairs_over_threshold"] - st["seg_ids"]), np.float64(0.0))
    return {"rand_index": ri, "adjusted_rand_index": ari, "variation_of_information": vi,
            "fowlkes_mallows_index": fm, "edit_distance": edit}


def evaluate(seg, gt, size_threshold=1000) -> dict:
    """Segmentation.evaluate's dict (without its printed lines)."""
    return scores(statistics(*contingency_triples(seg, gt), size_threshold=size_threshold))
