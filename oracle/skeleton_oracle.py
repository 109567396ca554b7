"""`skeletonize` restated (reference chunkflow/plugins/skeletonize.py -> kimimaro.skeletonize): a TEASAR skeleton of every
object of a segmentation chunk.  kimimaro is not vendored in the reference, so this module states the project's own rules and
csrc/skeleton.cu follows them bit for bit.  These are NOT kimimaro's skeletons.

All arithmetic is float64 with every operation rounded on its own (Python floats; numpy element-wise operations are not fused).

1. DBF.  For a voxel of label L != 0: the Euclidean distance, in physical units, to the nearest voxel whose label is not L;
   everything outside the chunk counts as 0 and label 0 gets 0.  Three line passes (x, y, z).  On a line, a run [a, b) of
   one non-zero label sees its two outside neighbours a - 1 and b at distance 0, so
       d2(q) = min(F-envelope(q), ((q - a + 1) w)^2, ((b - q) w)^2)
   where the envelope is Felzenszwalb-Huttenlocher's lower envelope of the parabolas F(p) + ((q - p) w)^2 of the run's own
   sites p (x pass: no sites; y pass: F = the x pass; z pass: F = the y pass).  DBF = float32(sqrt(d2)).
2. Objects: 26-connected components of one non-zero label, minus the skip ids and those under `dust_threshold` voxels.
3. Root: the voxel with the largest DBF, ties to the smallest linear index.
4. PDRF(v) = pdrf_scale * t^e + 1, t = 1 - DBF(v) / DBF(root), t^e by repeated multiplication left to right.  A step u -> v
   costs len(u -> v) * PDRF(v); D is the least fixed point of D(root) = 0, D(v) = min_u D(u) + cost(u -> v) (Dijkstra here).
   Parent(v) is the neighbour attaining the minimum, ties to the smallest index.  Refused unless
   (pdrf_scale + 1) * diagonal step * chunk voxels * (1 + 2^-19) < 2^53 * the smallest voxel size: then D is finite and every
   step raises it, so every Parent chain ends at the root.
5. Rounds: the target is the valid voxel with the largest D (ties: smallest index); the path runs from it along Parent to the
   root or to the first voxel already on the skeleton (not included); every path voxel p invalidates the voxels v of the object
   with d2(v, p) <= r * r, r = scale * DBF(p) + const, d2 summed z, y, x.  Until no valid voxel remains.
6. Per label: vertices are the skeleton voxels in ascending index at (i + 0.5) * w as float32 x, y, z; radii the DBF; edges
   (v, Parent(v)) for every vertex but the roots, as uint32 rows sorted by v.
"""
from __future__ import annotations

import heapq

import numpy as np

DEFAULTS = dict(scale=4.0, const=500.0, pdrf_scale=100000.0, pdrf_exponent=4, dust_threshold=1000)
DTYPES = (np.uint32, np.int32, np.uint64, np.int64)


def as_ids(seg) -> np.ndarray:
    """The ids as uint64, signed ones by their bit pattern; refuses what the device refuses."""
    seg = np.asarray(seg)
    if seg.ndim != 3:
        raise ValueError(f"skeletonize takes a (z, y, x) segmentation, not {seg.ndim}-D")
    if seg.dtype.type not in DTYPES:
        raise TypeError(f"skeletonize takes uint32, int32, uint64 or int64 ids, not {seg.dtype}")
    if seg.size >= 2 ** 32:
        raise ValueError("skeletonize: the chunk must have fewer than 2^32 voxels")
    if seg.dtype.kind == "i":
        seg = seg.view(seg.dtype.str.replace("i", "u"))
    return np.ascontiguousarray(seg).astype(np.uint64)


def check_voxel_size(voxel_size) -> tuple:
    w = tuple(float(v) for v in voxel_size)
    if len(w) != 3 or not all(np.isfinite(v) and v > 0 for v in w):
        raise ValueError(f"the voxel size is three positive (z, y, x) numbers, not {voxel_size}")
    return w


def _intersect(F, p: int, q: int, w: float) -> float:
    """Where the parabolas of sites p < q meet (FH), in positions along the line."""
    qw, pw = float(q) * w, float(p) * w
    return ((F[q] + qw * qw) - (F[p] + pw * pw)) / ((w * w) * float(2 * (q - p)))


def _line(lab, F, w: float, out) -> None:
    """One line: lab the ids, F the previous pass (None for x), out the new squared distances."""
    n = len(lab)
    a = 0
    while a < n:
        b = a + 1
        while b < n and lab[b] == lab[a]:
            b += 1
        if lab[a] != 0:
            v = [a]
            if F is not None:
                for q in range(a + 1, b):
                    while len(v) > 1 and _intersect(F, v[-1], q, w) <= _intersect(F, v[-2], v[-1], w):
                        v.pop()
                    v.append(q)
            k = 0
            for q in range(a, b):
                lo, hi = float(q - a + 1) * w, float(b - q) * w
                best = min(lo * lo, hi * hi)
                if F is not None:
                    while k + 1 < len(v) and _intersect(F, v[k], v[k + 1], w) < q:
                        k += 1
                    t = float(q - v[k]) * w
                    best = min(best, F[v[k]] + t * t)
                out[q] = best
        else:
            out[a:b] = 0.0
        a = b


def squared_dbf(seg, voxel_size=(1, 1, 1)) -> np.ndarray:
    """float64 squared distance to the boundary (rule 1), before the square root."""
    ids = as_ids(seg)
    wz, wy, wx = check_voxel_size(voxel_size)
    Z, Y, X = ids.shape
    d2x = np.zeros(ids.shape, np.float64)
    for z in range(Z):
        for y in range(Y):
            _line(ids[z, y, :].tolist(), None, wx, d2x[z, y, :])
    d2y = np.zeros(ids.shape, np.float64)
    for z in range(Z):
        for x in range(X):
            col = np.empty(Y)
            _line(ids[z, :, x].tolist(), d2x[z, :, x].tolist(), wy, col)
            d2y[z, :, x] = col
    d2 = np.zeros(ids.shape, np.float64)
    for y in range(Y):
        for x in range(X):
            col = np.empty(Z)
            _line(ids[:, y, x].tolist(), d2y[:, y, x].tolist(), wz, col)
            d2[:, y, x] = col
    return d2


def distance_transform(seg, voxel_size=(1, 1, 1)) -> np.ndarray:
    """float32 DBF of every voxel (rule 1)."""
    return np.sqrt(squared_dbf(seg, voxel_size)).astype(np.float32)


OFFSETS = [(dz, dy, dx) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dz, dy, dx) != (0, 0, 0)]


def step_length(off, w) -> float:
    """Physical length of a neighbour offset, summed z, y, x (13 distinct values)."""
    a, b, c = float(abs(off[0])) * w[0], float(abs(off[1])) * w[1], float(abs(off[2])) * w[2]
    return float(np.sqrt((a * a + b * b) + c * c))


def pdrf(dbf_v: float, dbf_max: float, pdrf_scale: float, e: int) -> float:
    t = 1.0 - float(dbf_v) / float(dbf_max)
    p = t
    for _ in range(e - 1):
        p = p * t
    return float(pdrf_scale) * p + 1.0


def objects(ids: np.ndarray, skip_ids=(), dust_threshold: int = 1000):
    """Rule 2 -> [(label, ascending linear indices)], by label then first voxel."""
    from scipy import ndimage
    skip = {int(i) % 2 ** 64 for i in (skip_ids or ())}
    out = []
    flat = ids.ravel()
    for L in np.unique(flat):
        L = int(L)
        if L == 0 or L in skip:
            continue
        comp, n = ndimage.label(ids == L, structure=np.ones((3, 3, 3), bool))
        cf = comp.ravel()
        idx = np.flatnonzero(cf)
        order = np.argsort(cf[idx], kind="stable")
        idx, lab = idx[order], cf[idx][order]
        starts = np.flatnonzero(np.r_[True, lab[1:] != lab[:-1]])
        for s, e in zip(starts, np.r_[starts[1:], len(idx)]):
            if e - s >= dust_threshold:
                out.append((L, idx[s:e]))
    return out


def neighbours(i: int, shape):
    Z, Y, X = shape
    z, r = divmod(i, Y * X)
    y, x = divmod(r, X)
    for k, (dz, dy, dx) in enumerate(OFFSETS):
        zz, yy, xx = z + dz, y + dy, x + dx
        if 0 <= zz < Z and 0 <= yy < Y and 0 <= xx < X:
            yield k, (zz * Y + yy) * X + xx


def geodesic(idx, dbf_flat, shape, w, pdrf_scale, e):
    """Rules 3 and 4 for one object -> (root, {voxel: D}, {voxel: Parent}, {voxel: PDRF})."""
    members = set(int(i) for i in idx)
    vals = dbf_flat[idx]
    root = int(idx[int(np.argmax(vals))])
    dmax = float(dbf_flat[root])
    P = {i: pdrf(dbf_flat[i], dmax, pdrf_scale, e) for i in members}
    lens = [step_length(o, w) for o in OFFSETS]
    D = {root: 0.0}
    heap = [(0.0, root)]
    done = set()
    while heap:
        d, u = heapq.heappop(heap)
        if u in done:
            continue
        done.add(u)
        for k, v in neighbours(u, shape):
            if v in members and v not in done:
                c = d + lens[k] * P[v]
                if c < D.get(v, np.inf):
                    D[v] = c
                    heapq.heappush(heap, (c, v))
    parent = {}
    for v in members:
        if v == root:
            parent[v] = v
            continue
        best, bu = np.inf, None
        for k, u in neighbours(v, shape):
            if u in members:
                c = D[u] + lens[k] * P[v]
                if c < best or (c == best and u < bu):
                    best, bu = c, u
        parent[v] = bu
    return root, D, parent, P


def trace(idx, dbf_flat, D, parent, root, shape, w, scale, const):
    """Rule 5 for one object -> (skeleton voxels in the order they were added, rounds, paths)."""
    Z, Y, X = shape
    idx = np.asarray(idx, np.int64)
    order = sorted(idx.tolist(), key=lambda i: (-D[i], i))
    coords = np.stack(np.unravel_index(idx, shape), 1).astype(np.float64)
    pos = {int(i): k for k, i in enumerate(idx)}
    valid = np.ones(len(idx), bool)
    on, added, paths = set(), [], []
    cursor = 0
    while True:
        while cursor < len(order) and not valid[pos[order[cursor]]]:
            cursor += 1
        if cursor == len(order):
            break
        v, path = order[cursor], []
        while v not in on:
            path.append(v)
            on.add(v)
            if v == root:
                break
            v = parent[v]
        paths.append(path)
        added += path
        for p in path:
            r = float(scale) * float(dbf_flat[p]) + float(const)
            pz, py, px = np.unravel_index(p, shape)
            dz = (coords[:, 0] - float(pz)) * w[0]
            dy = (coords[:, 1] - float(py)) * w[1]
            dx = (coords[:, 2] - float(px)) * w[2]
            valid[((dz * dz + dy * dy) + dx * dx) <= r * r] = False
    return added, paths


def skeletonize(seg, voxel_size=(1, 1, 1), scale=4, const=500, pdrf_scale=100000, pdrf_exponent=4, dust_threshold=1000,
                skip_ids=None, stats=None) -> dict:
    """Rules 1-6 -> {label: (vertices float32 (N, 3) x y z, edges uint32 (M, 2), radii float32 (N,))}, labels ascending."""
    ids = as_ids(seg)
    w = check_voxel_size(voxel_size)
    check_params(scale, const, pdrf_scale, pdrf_exponent, dust_threshold, w, ids.size)
    dbf = distance_transform(ids, w).ravel()
    per_label = {}
    for L, idx in objects(ids, skip_ids, int(dust_threshold)):
        root, D, parent, _ = geodesic(idx, dbf, ids.shape, w, float(pdrf_scale), int(pdrf_exponent))
        added, paths = trace(idx, dbf, D, parent, root, ids.shape, w, scale, const)
        if stats is not None:
            stats.setdefault("paths", []).append([len(p) for p in paths])
        per_label.setdefault(L, []).extend((v, parent[v]) for v in added)
    out = {}
    for L in sorted(per_label):
        vox = sorted(per_label[L])
        v = np.array([a for a, _ in vox], np.int64)
        par = np.array([b for _, b in vox], np.int64)
        out[L] = (vertex_positions(v, ids.shape, w), _edges(v, par), dbf[v].astype(np.float32))
    return out


def _edges(v, par):
    keep = v != par
    return np.stack([np.searchsorted(v, v[keep]), np.searchsorted(v, par[keep])], 1).astype(np.uint32).reshape(-1, 2)


def vertex_positions(v, shape, w):
    z, y, x = np.unravel_index(np.asarray(v, np.int64), shape)
    return np.stack([(x + 0.5) * w[2], (y + 0.5) * w[1], (z + 0.5) * w[0]], 1).astype(np.float32).reshape(-1, 3)


def check_params(scale, const, pdrf_scale, pdrf_exponent, dust_threshold, voxel_size=(1.0, 1.0, 1.0), voxels=1) -> None:
    for name, v in (("scale", scale), ("const", const), ("pdrf_scale", pdrf_scale)):
        if not (np.isfinite(float(v)) and float(v) >= 0):
            raise ValueError(f"skeletonize: {name} is a finite number >= 0, not {v}")
    if isinstance(pdrf_exponent, bool) or int(pdrf_exponent) != pdrf_exponent or not 1 <= int(pdrf_exponent) <= 16:
        raise ValueError(f"skeletonize: pdrf_exponent is an integer from 1 to 16, not {pdrf_exponent}")
    if isinstance(dust_threshold, bool) or int(dust_threshold) != dust_threshold or int(dust_threshold) < 0:
        raise ValueError(f"skeletonize: dust_threshold is an integer >= 0, not {dust_threshold}")
    # Rule 4 needs D finite and strictly increasing along every step, so that every Parent chain ends at the root: a path has
    # fewer than `voxels` steps, each costing at most the diagonal step times pdrf_scale + 1, and below 2^53 times the smallest
    # voxel size half an ulp of D is less than the cheapest step (the smallest voxel size).
    w = check_voxel_size(voxel_size)
    diagonal = step_length((1, 1, 1), w)
    bound = (((float(pdrf_scale) + 1.0) * diagonal) * float(voxels)) * (1.0 + 2.0 ** -19)
    if not (np.isfinite(diagonal) and bound < 2.0 ** 53 * min(w)):
        raise ValueError("skeletonize: D must stay finite and strictly increasing: (pdrf_scale + 1) * diagonal step * chunk voxels * "
                         "(1 + 2^-19) must be below 2^53 * the smallest voxel size")
