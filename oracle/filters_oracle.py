"""numpy restatement of `gaussian-filter` and the median-filter plugin (DESIGN.md section 0, row f8) -- the rules the CUDA
kernels of csrc/filter_kernels.cuh follow, written so that every rounding step is visible:

* weights  ``radius = int(4 sigma + 0.5)``, ``w = exp(-0.5 / sigma**2 * x**2)`` for x = -radius..radius, ``w /= w.sum()``, float64
  (:func:`gaussian_weights`; the library takes these weights from Python, never computes them);
* one 1-D pass per axis in axis order, skipped where ``sigma <= 1e-15``; per element, in float64 with every operation rounded
  separately: ``t = x[i] * w[0]``, then for j = radius .. 1: ``t = t + (x[i-j] + x[i+j]) * w[j]``;
* boundaries: one index map per mode (:func:`fold`), shared by both filters;
* a cast to the array's dtype after every pass (uint8: truncation toward zero, float32: round to nearest); the next pass reads
  the cast values;
* median: the window of extent s spans offsets -(s//2) .. s-1-(s//2); the result is element V//2 of the sorted window of V
  voxels.

These equal ``scipy.ndimage.gaussian_filter`` (truncate 4, mode 'reflect') and ``scipy.ndimage.median_filter`` bit for bit on
uint8 and float32 (tests/test_filters_oracle.py checks it live).  NaN and the sign of a zero in a median tie are outside that
claim.
"""
import numpy as np

MAX_RADIUS = 64
MAX_WINDOW = 125
MODES = {"reflect": 0, "grid-mirror": 0, "nearest": 1, "mirror": 2, "wrap": 3, "grid-wrap": 3, "constant": 4,
         "grid-constant": 4}
DTYPES = (np.dtype(np.uint8), np.dtype(np.float32))


def check_dtype(dtype):
    if np.dtype(dtype) not in DTYPES:
        raise TypeError(f"the filters take uint8 or float32 chunks, not {np.dtype(dtype)}")


def gaussian_weights(sigma):
    """float64 weights w[0..radius] (w[0] the centre) of scipy's gaussian kernel at truncate 4."""
    sigma = float(sigma)
    radius = int(4.0 * sigma + 0.5)
    x = np.arange(-radius, radius + 1)
    w = np.exp(-0.5 / sigma ** 2 * x ** 2)
    w = w / w.sum()
    return np.ascontiguousarray(w[radius:])


def per_axis(value, ndim, what="sigma"):
    v = np.asarray(value, dtype=np.float64 if what == "sigma" else np.int64)
    if v.ndim == 0:
        return [v.item()] * ndim
    if v.size != ndim:
        raise RuntimeError("sequence argument must have length equal to input rank")
    return [x.item() for x in v.ravel()]


def axis_weights(sigma, ndim):
    """The weights of every axis (None: the axis has no pass); ValueError above the radius limit."""
    out = []
    for s in per_axis(sigma, ndim):
        if s <= 1e-15:
            out.append(None)
            continue
        w = gaussian_weights(s)
        if len(w) - 1 > MAX_RADIUS:
            raise ValueError(f"gaussian filter: radius {len(w) - 1} exceeds the limit of {MAX_RADIUS} (sigma <= 15.9)")
        out.append(w)
    return out


def fold(i, n, mode):
    """Index i of a line of n elements under ``mode`` (a MODES value) -> index in 0..n-1, or -1 for the constant 0."""
    i = np.asarray(i, dtype=np.int64)
    if mode == 0:     # reflect: d c b a | a b c d | d c b a, period 2n
        k = np.mod(i, 2 * n)
        return np.where(k >= n, 2 * n - 1 - k, k)
    if mode == 1:     # nearest
        return np.clip(i, 0, n - 1)
    if mode == 2:     # mirror: d c b | a b c d | c b a, period 2n - 2; one element mirrors onto itself
        if n == 1:
            return np.zeros_like(i)
        k = np.mod(i, 2 * n - 2)
        return np.where(k >= n, 2 * n - 2 - k, k)
    if mode == 3:     # wrap
        return np.mod(i, n)
    if mode == 4:     # constant
        return np.where((i >= 0) & (i < n), i, -1)
    raise ValueError(f"unknown mode {mode}")


def cast(t, dtype):
    if np.dtype(dtype) == np.uint8:
        return np.trunc(t).astype(np.uint8)   # C conversion: toward zero (t >= 0 here)
    return t.astype(np.float32)               # round to nearest


def correlate_pass(a, w, axis):
    """One 1-D pass of the symmetric weights w[0..r] along ``axis`` with reflect boundaries, cast to a.dtype."""
    n, r = a.shape[axis], len(w) - 1
    x = np.moveaxis(a, axis, -1).astype(np.float64)
    idx = np.arange(n)
    t = x * w[0]
    for j in range(r, 0, -1):
        t = t + (x[..., fold(idx - j, n, 0)] + x[..., fold(idx + j, n, 0)]) * w[j]
    return np.moveaxis(cast(t, a.dtype), -1, axis)


def gaussian_filter(a, sigma):
    """scipy.ndimage.gaussian_filter(a, sigma) at its defaults, for uint8 / float32 ``a`` of any rank."""
    a = np.asarray(a)
    check_dtype(a.dtype)
    out = a.copy()
    for axis, w in enumerate(axis_weights(sigma, a.ndim)):
        if w is not None:
            out = correlate_pass(out, w, axis)
    return out


def gaussian_filter_2d(array, sigma):
    """Chunk.gaussian_filter_2d / the `gaussian-filter` command: for every z, gaussian_filter(array[..., z, :, :], sigma) --
    on a (c, z, y, x) chunk the section is (c, y, x), so the blur also runs across the channels."""
    out = np.array(array, copy=True)
    for z in range(out.shape[-3]):
        out[..., z, :, :] = gaussian_filter(out[..., z, :, :], sigma)
    return out


def gaussian_plugin(array, sigma=1.0):
    """plugins/gaussian_filter.execute: a 2-D (y, x) filter of every (channel,) z section."""
    out = np.array(array, copy=True)
    if out.ndim not in (3, 4):
        raise ValueError(f"only support 4 or 3d, but got {out.ndim}")
    flat = out.reshape((-1,) + out.shape[-2:])
    for k in range(flat.shape[0]):
        flat[k] = gaussian_filter(flat[k], sigma)
    return out


def median_filter(a, size=(3, 1, 1), mode="reflect"):
    """scipy.ndimage.median_filter(a, size=size, mode=mode) (cval 0, origin 0)."""
    a = np.asarray(a)
    check_dtype(a.dtype)
    if mode not in MODES:
        raise RuntimeError(f"boundary mode not supported: {mode}")
    sizes = per_axis(size, a.ndim, "size")
    if min(sizes) < 1:
        raise ValueError("every window extent must be at least 1")
    volume = int(np.prod(sizes))
    if volume > MAX_WINDOW:
        raise ValueError(f"median filter: a window of {volume} elements exceeds the limit of {MAX_WINDOW} (5x5x5)")
    m = MODES[mode]
    padded = np.concatenate([a.ravel(), np.zeros(1, a.dtype)])   # index -1: the constant 0
    coords = np.indices(a.shape)
    strides = [int(np.prod(a.shape[d + 1:])) for d in range(a.ndim)]
    window = []
    for offs in np.ndindex(*sizes):
        idx = np.zeros(a.shape, np.int64)
        outside = np.zeros(a.shape, bool)
        for d, o in enumerate(offs):
            k = fold(coords[d] + o - sizes[d] // 2, a.shape[d], m)
            outside |= k < 0
            idx += np.where(k < 0, 0, k) * strides[d]
        window.append(np.where(outside, -1, idx))
    vals = padded[np.stack(window)]
    return np.sort(vals, axis=0)[volume // 2]
