"""CPU oracle for ``agglomerate`` with waterz's histogram-quantile scoring functions (TEST INFRASTRUCTURE).

Scoring function: ``OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B[, I]>>`` -- lsd's ``hist_quant_50``
is Q = 50, B = 256, I = false, and ``hist_quant_50_initmax`` the same with I = true.  Everything else (watershed fragments,
the faces between fragments, the flip of chunkflow's channel order, the merge loop's stop rule and surviving ids) is as in
``oracle/agglomeration_oracle.py``.

PARITY UNPINNED: waterz (github.com/funkey/waterz, a Cython/C++ package; the reference does not pin a version and does not
list it in requirements.txt) is neither vendored in /root/reference nor installed in this image, and the reference holds no
test or golden vector for this plugin.  This file restates the rules below; the native library matches it bit for bit.

  1. bin of a face affinity ``a``: float32, clamped to [0, 1], NaN as 0 (as for the mean); bin = min(int(a * B), B - 1),
     the product in float32.
  2. histogram of an edge: per bin, the number of faces between the two fragments (the faces and channels of
     ``agglomeration_oracle.region_graph``).  With I = true the edge also carries the largest clamped face affinity (float32).
  3. quantile: n = the histogram's total, pivot = min(floor(Q n / 100) + 1, n); the quantile bin is the first bin whose
     cumulative count reaches the pivot, its value (bin + 0.5) / B, and the score 1 - value (double).
  4. I = true: an edge never POOLED (two edges to a common neighbour combined by a merge) scores 1 - its maximum (double);
     once pooled it scores from its histogram as in 3.  An edge only MOVED to the merged cluster keeps its score.  I
     omitted means true (waterz's declared default, as restated here).
  5. loop: merge the edge of the smallest (score, anchor) until that score reaches the threshold; the merged cluster keeps
     the smaller id; a pooled edge's histogram is the bin-wise sum of the two.
  6. anchor of a pooled edge: the anchor of whichever of the two pooled edges comes first in (score, anchor) order (the
     mean keeps the smaller anchor).  An original edge's anchor is its (u << 32 | v).
"""
import heapq

import numpy as np

from oracle.agglomeration_oracle import watershed


def affinity_bins(a: np.ndarray, bins: int) -> np.ndarray:
    """Rule 1: the bin of every affinity (int64) -- and, for rule 2, the clamped affinities themselves (float32)."""
    a = np.asarray(a, np.float32)
    with np.errstate(invalid="ignore"):
        c = np.where(a > 0, np.minimum(a, np.float32(1)), np.float32(0)).astype(np.float32)
    b = np.minimum((c * np.float32(bins)).astype(np.int64), bins - 1)
    return b, c


def region_graph_histograms(affs: np.ndarray, fragments: np.ndarray, B: int, with_max: bool):
    """(u, v, offsets, bins, counts, maxima): edges sorted by (u, v), u < v; edge i holds bins[offsets[i]:offsets[i+1]]
    (uint8, increasing) with their counts (uint32); maxima (float32) when ``with_max``, else None."""
    affs = np.asarray(affs, np.float32)
    frag = np.asarray(fragments).astype(np.int64)
    keys, vals = [], []
    for c in range(3):
        hi = [slice(None)] * 3
        lo = [slice(None)] * 3
        hi[c], lo[c] = slice(1, None), slice(None, -1)
        a, b = frag[tuple(hi)], frag[tuple(lo)]
        sel = (a != 0) & (b != 0) & (a != b)
        u, v = np.minimum(a[sel], b[sel]), np.maximum(a[sel], b[sel])
        keys.append((u << 32) | v)
        vals.append(affs[c][tuple(hi)][sel])
    keys, vals = np.concatenate(keys), np.concatenate(vals)
    uniq, inv = np.unique(keys, return_inverse=True)
    b, clamped = affinity_bins(vals, B)
    pair_bin, counts = np.unique(inv.astype(np.int64) * 256 + b, return_counts=True)
    edge = pair_bin // 256
    offsets = np.zeros(len(uniq) + 1, np.uint64)
    np.add.at(offsets, edge + 1, 1)
    offsets = np.cumsum(offsets).astype(np.uint64)
    maxima = None
    if with_max:
        maxima = np.zeros(len(uniq), np.float32)
        np.maximum.at(maxima, inv, clamped)
    return ((uniq >> 32).astype(np.uint32), (uniq & 0xFFFFFFFF).astype(np.uint32), offsets, (pair_bin % 256).astype(np.uint8),
            counts.astype(np.uint32), maxima)


def quantile_score(hist: np.ndarray, Q: int, B: int) -> float:
    """Rule 3 for a dense histogram of B bins."""
    n = int(hist.sum())
    pivot = min(Q * n // 100 + 1, n)
    b = int(np.searchsorted(np.cumsum(hist), pivot))   # the first bin whose cumulative count >= pivot
    return 1.0 - (b + 0.5) / B


def agglomerate_edges_quantile(num_nodes: int, u, v, offsets, bins, counts, maxima, threshold: float, Q: int, B: int,
                               init_with_max: bool) -> np.ndarray:
    """root_of (num_nodes,) uint32, rules 3-6: a global heap of (score, anchor) with lazy deletion.  Every state of an edge
    gets a new serial number; a heap entry whose serial is not the edge's any more is stale."""
    adj = [dict() for _ in range(num_nodes)]
    heap = []
    offsets = np.asarray(offsets).astype(np.int64)
    serial = 0
    for i, (a, b) in enumerate(zip(np.asarray(u).tolist(), np.asarray(v).tolist())):
        a, b = min(a, b), max(a, b)
        hist = np.zeros(B, np.int64)
        sl = slice(offsets[i], offsets[i + 1])
        hist[np.asarray(bins)[sl].astype(np.int64)] = np.asarray(counts)[sl]
        sc = 1.0 - float(np.float32(maxima[i])) if init_with_max else quantile_score(hist, Q, B)
        anchor = (a << 32) | b
        rec = (sc, anchor, hist, serial)
        adj[a][b] = adj[b][a] = rec
        heap.append((sc, anchor, a, b, serial))
        serial += 1
    heapq.heapify(heap)
    alive = [True] * num_nodes
    parent = list(range(num_nodes))
    thr = float(np.float32(threshold))
    while heap:
        sc, anchor, a, b, ser = heapq.heappop(heap)
        if not (alive[a] and alive[b]) or b not in adj[a] or adj[a][b][3] != ser:
            continue   # stale
        if not sc < thr:
            break
        alive[b] = False        # b (the larger id) is merged into a
        parent[b] = a
        del adj[a][b]
        for n, rec in adj[b].items():
            if n == a:
                continue
            del adj[n][b]
            if n in adj[a]:      # pooled: histograms add, score from the histogram, anchor of the first key (rule 6)
                so, ao, ho, _ = adj[a][n]
                sn, an, hn, _ = rec
                hist = ho + hn
                first = min((so, ao), (sn, an))
                rec = (quantile_score(hist, Q, B), first[1], hist, serial)
                serial += 1
            adj[a][n] = adj[n][a] = rec   # moved: keeps its score, anchor and serial
            heapq.heappush(heap, (rec[0], rec[1], min(a, n), max(a, n), rec[3]))
        adj[b] = {}
    out = np.zeros(num_nodes, np.uint32)
    for i in range(num_nodes):
        r = i
        while parent[r] != r:
            r = parent[r]
        out[i] = r
    return out


def agglomerate(affs: np.ndarray, threshold: float, Q: int, B: int, init_with_max: bool, fragments=None,
                aff_threshold_low: float = 0.001, aff_threshold_high: float = 0.9999, flip_channel: bool = True) -> np.ndarray:
    """``plugins/agglomerate.py: execute`` with a histogram-quantile scoring function -> (z, y, x) uint64 segmentation."""
    affs = np.asarray(affs)
    if flip_channel:
        affs = np.flip(affs, axis=0)
    affs = np.ascontiguousarray(affs, dtype=np.float32)
    if fragments is None:
        fragments = watershed(affs, aff_threshold_low, aff_threshold_high)
    fragments = np.asarray(fragments)
    num_nodes = int(fragments.max()) + 1 if fragments.size else 1
    u, v, off, bins, counts, mx = region_graph_histograms(affs, fragments, B, init_with_max)
    root = agglomerate_edges_quantile(num_nodes, u, v, off, bins, counts, mx, threshold, Q, B, init_with_max)
    return root[fragments].astype(np.uint64)
