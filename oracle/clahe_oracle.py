"""numpy restatement of `clahe` (DESIGN.md section 0, row f9) -- ``cv2.createCLAHE(clipLimit, tileGridSize).apply`` on uint8
sections, which the reference's plugin ``plugins/clahe.py`` runs on every z -- written so that every rounding step is visible.
The CUDA kernels of csrc/clahe_kernels.cuh follow these rules:

* padding: none when ``W % tiles_x == 0`` and ``H % tiles_y == 0``; otherwise ``tiles_y - H % tiles_y`` rows at the bottom and
  ``tiles_x - W % tiles_x`` columns at the right (a whole tile row or column even where that axis divides: OpenCV's rule),
  reflected without repeating the edge (BORDER_REFLECT_101, numpy 'reflect', repeated where the pad is longer than the section);
  tiles of ``th = padded_H / tiles_y`` by ``tw = padded_W / tiles_x`` pixels, ``T = th * tw``;
* clip limit: ``cl = max(int(clip_limit * T / 256), 1)`` in float64, the cast truncating (x86: a value out of the int32 range
  becomes INT32_MIN, so cl = 1); no clipping where ``clip_limit <= 0``;
* per tile, on the 256-bin histogram of the padded tile: ``clipped = sum(max(h - cl, 0))``, ``h = min(h, cl)``, every bin gets
  ``clipped // 256`` more, and bins 0, step, 2 step, ... one more each while ``clipped % 256`` lasts,
  ``step = max(256 // (clipped % 256), 1)``;
* LUT: ``lut[v] = sat_u8(rint(float32(cumsum[v]) * (float32(255) / float32(T))))``, rint halves to even;
* interpolation in float32, every multiply and add rounded on its own: ``txf = x * (1 / tw) - 0.5``, ``tx1 = floor(txf)``,
  ``xa = txf - tx1``, ``xa1 = 1 - xa``, ``tx2 = min(tx1 + 1, tiles_x - 1)`` from the unclamped tx1, then ``tx1 = max(tx1, 0)``;
  the same along y; ``res = (L11 xa1 + L12 xa) ya1 + (L21 xa1 + L22 xa) ya``; out ``sat_u8(rint(res))``.

``fma=True`` contracts every ``a * b + c`` of the interpolation into one rounding; it is a negative control only (the golden
vectors differ from it), showing that the separate roundings matter.
"""
import numpy as np

BINS = 256
INT32_MIN = -2 ** 31


def check(array, tile_grid_size):
    """The refusals: uint8 only (TypeError), (z, y, x) only and tiles >= 1 (ValueError)."""
    if np.asarray(array).dtype != np.uint8:
        raise TypeError(f"clahe takes uint8 images, not {np.asarray(array).dtype}")
    if np.ndim(array) != 3:
        raise ValueError(f"clahe takes a (z, y, x) image, not {np.ndim(array)} dimensions")
    tx, ty = (int(v) for v in tile_grid_size)
    if tx < 1 or ty < 1:
        raise ValueError(f"the tile grid {tile_grid_size} has fewer than one tile along an axis")
    return tx, ty


def geometry(h, w, tiles_x, tiles_y):
    """(padded_h, padded_w, th, tw)"""
    if w % tiles_x == 0 and h % tiles_y == 0:
        ph, pw = h, w
    else:
        ph, pw = h + tiles_y - h % tiles_y, w + tiles_x - w % tiles_x
    return ph, pw, ph // tiles_y, pw // tiles_x


def clip_count(clip_limit, tile_pixels):
    """cl, or None where there is no clipping."""
    if not clip_limit > 0:
        return None
    c = float(clip_limit) * tile_pixels / BINS
    cl = int(c) if -2.0 ** 31 < c < 2.0 ** 31 else INT32_MIN
    return max(cl, 1)


def tile_luts(padded, tiles_x, tiles_y, cl):
    """(tiles_y, tiles_x, 256) uint8 LUTs of a padded section, built a few tile rows at a time."""
    ph, pw = padded.shape
    th, tw = ph // tiles_y, pw // tiles_x
    scale = np.float32(255) / np.float32(th * tw)
    i = np.arange(BINS)
    out = np.empty((tiles_y, tiles_x, BINS), np.uint8)
    rows = max(1, 4096 // tiles_x)
    for y0 in range(0, tiles_y, rows):
        ny = min(rows, tiles_y - y0)
        t = padded[y0 * th:(y0 + ny) * th].reshape(ny, th, tiles_x, tw).transpose(0, 2, 1, 3).reshape(ny, tiles_x, th * tw)
        tiles = np.arange(ny * tiles_x).reshape(ny, tiles_x, 1) * BINS
        hist = np.bincount((tiles + t).ravel(), minlength=tiles.size * BINS).reshape(ny, tiles_x, BINS)
        if cl is not None:
            clipped = np.maximum(hist - cl, 0).sum(-1, keepdims=True)
            residual = clipped % BINS
            step = np.maximum(BINS // np.maximum(residual, 1), 1)
            hist = np.minimum(hist, cl) + clipped // BINS + ((i % step == 0) & (i // step < residual))
        lut = np.rint(np.cumsum(hist, -1).astype(np.float32) * scale)
        out[y0:y0 + ny] = np.clip(lut, 0, 255)
    return out


def _axis(n, tiles, size, fma):
    """(t1, t2, a, a1) float32 coordinates of positions 0..n-1 along one axis of `tiles` tiles of `size` pixels."""
    inv = np.float32(1.0) / np.float32(size)
    pos = np.arange(n, dtype=np.float32)
    f = (pos.astype(np.float64) * np.float64(inv) - 0.5).astype(np.float32) if fma else pos * inv - np.float32(0.5)
    t1 = np.floor(f).astype(np.int64)
    a = f - t1.astype(np.float32)
    a1 = np.float32(1) - a
    t2 = np.minimum(t1 + 1, tiles - 1)
    return np.maximum(t1, 0), t2, a, a1


def apply_section(sec, clip_limit=40.0, tile_grid_size=(8, 8), fma=False):
    """cv2.createCLAHE(clip_limit, tile_grid_size).apply(sec) for one (y, x) uint8 section."""
    tiles_x, tiles_y = (int(v) for v in tile_grid_size)
    h, w = sec.shape
    ph, pw, th, tw = geometry(h, w, tiles_x, tiles_y)
    padded = np.pad(sec, ((0, ph - h), (0, pw - w)), mode="reflect")
    lut = tile_luts(padded, tiles_x, tiles_y, clip_count(clip_limit, th * tw))
    tx1, tx2, xa, xa1 = _axis(w, tiles_x, tw, fma)
    ty1, ty2, ya, ya1 = _axis(h, tiles_y, th, fma)
    v = sec.astype(np.int64)
    L = lambda ty, tx: lut[ty[:, None], tx[None, :], v].astype(np.float32)
    L11, L12, L21, L22 = L(ty1, tx1), L(ty1, tx2), L(ty2, tx1), L(ty2, tx2)
    ya, ya1 = ya[:, None], ya1[:, None]
    if fma:   # each a * b + c rounded once
        f64 = lambda a: a.astype(np.float64)
        top = (f64(L11 * xa1) + f64(L12) * xa).astype(np.float32)
        bot = (f64(L21 * xa1) + f64(L22) * xa).astype(np.float32)
        res = (f64(top * ya1) + f64(bot) * ya).astype(np.float32)
    else:
        res = (L11 * xa1 + L12 * xa) * ya1 + (L21 * xa1 + L22 * xa) * ya
    return np.clip(np.rint(res), 0, 255).astype(np.uint8)


def clahe(array, clip_limit=20.0, tile_grid_size=(512, 512), fma=False):
    """The reference plugin on a (z, y, x) uint8 image: every section on its own.  tile_grid_size is (x, y), cv2's order."""
    check(array, tile_grid_size)
    return np.stack([apply_section(s, clip_limit, tile_grid_size, fma) for s in np.asarray(array)])
