"""numpy restatement of `downsample` (DESIGN.md section 0, row f7), written from the rules of the reference's vendored
downsampler (reference lib/igneous/downsample.py) and its `downsample` command (flow/flow.py:1545-1573).  Pinned to the real
module by tests/golden/downsample_reference.npz and, where the reference tree exists, live (oracle/downsample_harness.py).
tinybrain, which the command calls, is a third-party package outside the reference tree: PARITY UNPINNED.

* averaging (uint8): floor(block sum / voxels in the block), blocks clipped at the far edges, output ceil(shape / factor);
* segmentation: the level plan of :func:`plan` -- countless3d, countless2d or striding per level, ``factor // 2`` between
  levels (the reference's ``factor / 2`` raises on every second level);
* countless2d: a if a == b or a == c, else b if b == c, else d; an odd side gets a copy of its first plane in front;
* countless3d: the first value seen >= 4 times, else >= 3, else >= 2 times among voxels 0..6, else voxel 7;
* the all-ones id (max of an unsigned type, -1 of a signed one) never counts as a pick in countless3d, nor in countless2d
  for types the reference does not widen (64-bit and signed ones).
"""
import numpy as np

STRIDE, COUNTLESS2D, COUNTLESS3D = "stride", "countless2d", "countless3d"
MAX_AVERAGE_BLOCK = 65793
MAX_FACTOR_PRODUCT = 2 ** 31 - 1


def _factor(factor):
    f = tuple(int(v) for v in factor)
    if len(f) != 3:
        raise ValueError(f"the factor is (z, y, x), not {f}")
    if min(f) <= 0:
        raise ValueError(f"Factors less than one don't make sense. Factor: {f}")
    return f


def _pow2(v):
    return v > 0 and v & (v - 1) == 0


def plan(dtype, shape, factor):
    """[(algorithm, factor of the level, preserved axis or None, output shape)] of downsample_segmentation; [] when the input
    is the result.  ValueError for the factors on which the reference (with factor // 2) raises."""
    f, s = _factor(factor), tuple(int(v) for v in shape)
    if f[0] * f[1] * f[2] > MAX_FACTOR_PRODUCT:
        raise ValueError("the factor's product exceeds 2^31 - 1")
    integer = np.dtype(dtype).kind in "ui"
    levels = []
    while True:
        if min(f) <= 0:
            raise ValueError(f"the factor's recursion reaches {f}: a factor of 0 on an axis with factor 1")
        if f == (1, 1, 1):
            return levels
        pot, has_one = all(_pow2(v) for v in f), 1 in f
        if integer and pot and not has_one and all(v % 2 == 0 for v in s):
            s = tuple(v // 2 for v in s)
            levels.append((COUNTLESS3D, f, None, s))
            f = tuple(v // 2 for v in f)
            continue
        if not integer or not (pot and has_one):
            levels.append((STRIDE, f, None, tuple(-(-a // b) for a, b in zip(s, f))))
            return levels
        p = f.index(1)
        s = tuple(v if i == p else (v + 1) // 2 for i, v in enumerate(s))
        levels.append((COUNTLESS2D, f, p, s))
        f = tuple(1 if i == p else v // 2 for i, v in enumerate(f))


def downsample_with_averaging(a, factor):
    """uint8 (z, y, x) -> uint8 ceil(shape / factor)."""
    a = np.asarray(a)
    assert a.dtype == np.uint8 and a.ndim == 3
    f = _factor(factor)
    if f[0] * f[1] * f[2] > MAX_AVERAGE_BLOCK:
        raise ValueError("averaging blocks of more than 65793 voxels are refused")
    if f == (1, 1, 1):
        return a.copy()
    o = tuple(-(-s // k) for s, k in zip(a.shape, f))
    padded = np.zeros(tuple(n * k for n, k in zip(o, f)), np.uint32)
    padded[:a.shape[0], :a.shape[1], :a.shape[2]] = a
    sums = padded.reshape(o[0], f[0], o[1], f[1], o[2], f[2]).sum(axis=(1, 3, 5), dtype=np.uint64)
    counts = [np.minimum(np.arange(n) * k + k, s) - np.arange(n) * k for n, k, s in zip(o, f, a.shape)]
    count = counts[0][:, None, None] * counts[1][None, :, None] * counts[2][None, None, :]
    return (sums // count.astype(np.uint64)).astype(np.uint8)


def _all_ones(dtype):
    return np.array(-1).astype(dtype) if np.dtype(dtype).kind == "i" else np.array(np.iinfo(dtype).max, dtype)


def _widened(dtype):
    """countless2d widens uint8 / uint16 / uint32 before offsetting the ids: every id counts."""
    return np.dtype(dtype) in (np.dtype(np.uint8), np.dtype(np.uint16), np.dtype(np.uint32))


def _pairs(n):
    j = np.arange((n + 1) // 2)
    odd = n % 2
    return np.maximum(2 * j - odd, 0), 2 * j + 1 - odd


def countless2d(a, preserved):
    axes = [i for i in range(3) if i != preserved]
    lo_u, hi_u = _pairs(a.shape[axes[0]])
    lo_v, hi_v = _pairs(a.shape[axes[1]])
    u_lo, u_hi = np.take(a, lo_u, axis=axes[0]), np.take(a, hi_u, axis=axes[0])
    va, vb = np.take(u_lo, lo_v, axis=axes[1]), np.take(u_lo, hi_v, axis=axes[1])
    vc, vd = np.take(u_hi, lo_v, axis=axes[1]), np.take(u_hi, hi_v, axis=axes[1])
    if _widened(a.dtype):
        ca = cb = True
    else:
        ones = _all_ones(a.dtype)
        ca, cb = va != ones, vb != ones
    return np.where(ca & ((va == vb) | (va == vc)), va, np.where(cb & (vb == vc), vb, vd))


def countless3d(a):
    assert all(s % 2 == 0 for s in a.shape)
    v = [a[dz::2, dy::2, dx::2] for dz in range(2) for dy in range(2) for dx in range(2)]   # i = 4 dz + 2 dy + dx
    valid = [x != _all_ones(a.dtype) for x in v]
    count = [sum((v[i] == v[j]).astype(np.int8) for j in range(8)) for i in range(8)]
    count7 = [sum((v[i] == v[j]).astype(np.int8) for j in range(7)) for i in range(7)]
    out = v[7].copy()
    done = np.zeros(v[0].shape, bool)
    for rank_counts, r, n in ((count, 4, 8), (count, 3, 8), (count7, 2, 7)):
        for i in range(n):
            take = ~done & valid[i] & (rank_counts[i] >= r)
            out[take] = v[i][take]
            done |= take
    return out


def stride(a, factor):
    return a[::factor[0], ::factor[1], ::factor[2]].copy()


def downsample_segmentation(a, factor):
    """Integer or boolean (z, y, x) -> the same dtype, level after level."""
    a = np.asarray(a)
    assert a.ndim == 3
    out = a
    for algo, f, preserved, _ in plan(a.dtype, a.shape, factor):
        if algo == COUNTLESS3D:
            out = countless3d(out)
        elif algo == COUNTLESS2D:
            out = countless2d(out, preserved)
        else:
            out = stride(out, f)
    return out.copy() if out is a else out


def is_image(a):
    return a.ndim == 3 and a.dtype == np.uint8


def is_segmentation(a):
    return a.ndim == 3 and (np.issubdtype(a.dtype, np.integer) or a.dtype == bool) and a.dtype != np.uint8


def downsample(a, factor=(2, 2, 2)):
    """The `downsample` command's dispatch on the (z, y, x) array."""
    a = np.asarray(a)
    if is_image(a):
        return downsample_with_averaging(a, factor)
    if is_segmentation(a):
        return downsample_segmentation(a, factor)
    raise TypeError(f'only support image or segmentation, but got: {a.dtype}')


def thumbnail(affinity, mips=6):
    """The thumbnail pyramid of `save-precomputed --create-thumbnail` restated on the (z, y, x) side: the last channel as
    uint8 (`quantize --mode z`), then ``mips`` levels of averaging by (1, 2, 2).  -> [level 1, ..., level mips]."""
    image = (np.asarray(affinity)[-1] * np.float32(255)).astype(np.uint8)
    out = []
    for _ in range(mips):
        image = downsample_with_averaging(image, (1, 2, 2))
        out.append(image)
    return out
