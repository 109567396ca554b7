// Device code of `clahe` (DESIGN.md section 0, row f9), included by clahe.cu (which tests/host_emulation also compiles for
// the host, behind a one-lane CUDA shim).  The arithmetic is OpenCV's cv2.createCLAHE(clip, (tiles_x, tiles_y)).apply on
// uint8 sections, which the reference's plugins/clahe.py runs on every z, restated in oracle/clahe_oracle.py:
//   tiles      th x tw pixels of the section padded at the bottom and right (BORDER_REFLECT_101: flt_fold kFltMirror), the
//              padded section never materialised: a tile reads its rows and columns through the index map;
//   tile LUT   256-bin histogram h, clipped at cl and redistributed: h = min(h, cl) + batch, plus one at bins 0, step, ...
//              while the residual lasts; lut[v] = sat_u8(rint(float(cumsum(v)) * (255.f / T)));
//              cumsum(v) = sum_{i <= v} min(h[i], cl) + batch (v + 1) + (residual ? min(residual, v / step + 1) : 0);
//   output     the float32 bilinear blend of the 4 neighbouring tiles' LUTs at the pixel's value, every multiply and add
//              rounded on its own (__fmul_rn / __fadd_rn: nvcc would contract a * b + c into an FMA, and cv2 does not).
// Two paths, selected from T = th * tw (clahe_small_tiles):
//   table       T > kClaheSmallTileMax: clahe_lut_kernel, one CTA per (tile, section), builds the tile's histogram in
//               lane-private shared sub-histograms and writes its 256-byte LUT to the workspace; clahe_table_kernel, one CTA
//               per (tile, section), stages the 3 x 3 LUTs around its tile in shared memory and writes the tile's pixels.
//               Sections go in batches whose LUTs fit kClaheWorkspaceTarget.
//   small tile  T <= kClaheSmallTileMax: clahe_small_kernel, one CTA per region of tiles, stages the raw pixels of the region's
//               tiles and of the ring of tiles around it, and evaluates each neighbour's LUT at the pixel's value from the
//               closed form above: no table, no workspace, one launch for the chunk.
// Both read every output pixel's input once and write it once, 16 bytes at a time where the output row is aligned.  Every
// index is 64-bit; the input and output never overlap.
#include "fold.cuh"

constexpr int kClaheBins = 256;
constexpr int kClaheThreads = 256;
constexpr int64_t kClaheSmallTileMax = 64;   // measured on an H100: the small-tile path is 2x faster at T = 64, 2x slower at T = 128
constexpr int64_t kClaheWorkspaceTarget = 32ll << 20;
constexpr int64_t kClaheMaxSide = 1ll << 24;   // float(x) is exact below 2^24
constexpr int kClaheSmallSmem = 48 << 10;

struct ClaheGeom {
  int64_t H, W;                  // section
  int64_t tiles_x, tiles_y, th, tw;
  int64_t T;                     // th * tw
  int64_t cl;                    // clip count (INT64_MAX: no clipping)
  float lut_scale, inv_th, inv_tw;
};

// cv2's arithmetic on the host: 1 / tw, 255 / T in float32, the clip count in float64 (x86 turns an out-of-range cast into
// INT32_MIN, so such a clip limit clips at 1).
inline ClaheGeom clahe_geometry(int64_t H, int64_t W, int64_t tiles_x, int64_t tiles_y, double clip_limit) {
  ClaheGeom g{};
  g.H = H;
  g.W = W;
  g.tiles_x = tiles_x;
  g.tiles_y = tiles_y;
  const bool pad = W % tiles_x != 0 || H % tiles_y != 0;
  g.th = (pad ? H + tiles_y - H % tiles_y : H) / tiles_y;
  g.tw = (pad ? W + tiles_x - W % tiles_x : W) / tiles_x;
  g.T = g.th * g.tw;
  g.cl = INT64_MAX;
  if (clip_limit > 0) {
    const double c = clip_limit * (double)g.T / kClaheBins;
    const int64_t cl = (c > -2147483649.0 && c < 2147483648.0) ? (int64_t)c : INT32_MIN;
    g.cl = cl < 1 ? 1 : cl;
  }
  g.lut_scale = 255.0f / (float)g.T;
  g.inv_th = 1.0f / (float)g.th;
  g.inv_tw = 1.0f / (float)g.tw;
  return g;
}

inline bool clahe_small_tiles(const ClaheGeom& g) { return g.T <= kClaheSmallTileMax; }

__host__ __device__ __forceinline__ int64_t clahe_min(int64_t a, int64_t b) { return a < b ? a : b; }
__host__ __device__ __forceinline__ int64_t clahe_max(int64_t a, int64_t b) { return a < b ? b : a; }

// The redistribution of `clipped` counts: batch to every bin, one more to bins 0, step, ... while the residual lasts.
struct ClaheSpread {
  int64_t batch;
  int residual, step;
};

__device__ __forceinline__ ClaheSpread clahe_spread(int64_t clipped) {
  ClaheSpread s;
  s.batch = clipped / kClaheBins;
  s.residual = (int)(clipped % kClaheBins);
  s.step = s.residual ? (kClaheBins / s.residual > 1 ? kClaheBins / s.residual : 1) : 1;
  return s;
}

// lut[v] from sum_{i <= v} min(h[i], cl); every increment of the residual loop lands, since (residual - 1) step < 256.
__device__ __forceinline__ int clahe_lut_value(int64_t kept, int v, const ClaheSpread& s, float scale) {
  const int64_t cum = kept + s.batch * (v + 1) + (s.residual ? (s.residual < v / s.step + 1 ? s.residual : v / s.step + 1) : 0);
  const int q = __float2int_rn(__fmul_rn((float)cum, scale));
  return q < 0 ? 0 : q > 255 ? 255 : q;
}

// One axis of the blend at position p: the slot of tile t1 (unclamped) relative to the first staged tile `base`, and the
// weights.  The staged slot k holds tile clamp(base + k), which is cv2's max(t1, 0) and min(t1 + 1, tiles - 1).
struct ClaheAxis {
  int64_t slot;
  float a, a1;
};

__device__ __forceinline__ ClaheAxis clahe_axis(int64_t p, float inv, int64_t base) {
  const float f = __fadd_rn(__fmul_rn((float)p, inv), -0.5f);
  const float t1 = floorf(f);
  ClaheAxis r;
  r.slot = (int64_t)t1 - base;
  r.a = __fsub_rn(f, t1);
  r.a1 = __fsub_rn(1.0f, r.a);
  return r;
}

__device__ __forceinline__ uint8_t clahe_blend(float l11, float l12, float l21, float l22, const ClaheAxis& y, const ClaheAxis& x) {
  const float top = __fadd_rn(__fmul_rn(l11, x.a1), __fmul_rn(l12, x.a));
  const float bottom = __fadd_rn(__fmul_rn(l21, x.a1), __fmul_rn(l22, x.a));
  const int q = __float2int_rn(__fadd_rn(__fmul_rn(top, y.a1), __fmul_rn(bottom, y.a)));
  return (uint8_t)(q < 0 ? 0 : q > 255 ? 255 : q);
}

// Writes the pixels [y0, y1) x [x0, x1) of one section; lut(sy, sx, v) is the LUT of staged slot (sy, sx) at value v, the
// slots counted from tile (ty_base, tx_base).  Work items are 16-byte groups of the output row: a whole group is stored as
// one uint4 (and loaded as one where the input is aligned too), a partial one byte by byte.
template <typename Lut>
__device__ __forceinline__ uint8_t clahe_pixel(const Lut& lut, const ClaheGeom& g, const ClaheAxis& ay, int64_t x, int64_t tx_base, int v) {
  const ClaheAxis ax = clahe_axis(x, g.inv_tw, tx_base);
  return clahe_blend((float)lut(ay.slot, ax.slot, v), (float)lut(ay.slot, ax.slot + 1, v), (float)lut(ay.slot + 1, ax.slot, v),
                     (float)lut(ay.slot + 1, ax.slot + 1, v), ay, ax);
}

template <typename Lut>
__device__ __forceinline__ void clahe_write(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, const ClaheGeom& g,
                                            int64_t y0, int64_t y1, int64_t x0, int64_t x1, int64_t ty_base, int64_t tx_base,
                                            const Lut& lut) {
  // a row segment spans at most `groups` 16-byte groups; a tile or a region has fewer than 2^31 items (32-bit division)
  const unsigned int groups = (unsigned int)((x1 - x0 + 15) / 16 + 1), items = (unsigned int)(y1 - y0) * groups;
  for (unsigned int item = threadIdx.x; item < items; item += blockDim.x) {
    const int64_t y = y0 + item / groups, k = item % groups;
    const uint8_t* src = in + y * g.W;
    uint8_t* dst = out + y * g.W;
    const int64_t first = (int64_t)(reinterpret_cast<uintptr_t>(dst + x0) & ~(uintptr_t)15) - (int64_t)reinterpret_cast<uintptr_t>(dst);
    const int64_t xs = clahe_max(x0, first + 16 * k), xe = clahe_min(x1, first + 16 * k + 16);
    if (xs >= xe) continue;
    const ClaheAxis ay = clahe_axis(y, g.inv_th, ty_base);
    if (xe - xs == 16) {
      uint4 q;
      if ((reinterpret_cast<uintptr_t>(src + xs) & 15) == 0) {
        q = __ldg(reinterpret_cast<const uint4*>(src + xs));
      } else {
        unsigned int w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < 16; ++j) w[j >> 2] |= (unsigned int)__ldg(src + xs + j) << (8 * (j & 3));
        q = make_uint4(w[0], w[1], w[2], w[3]);
      }
      unsigned int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        unsigned int o = 0;
#pragma unroll 1
        for (int j = 0; j < 4; ++j) o |= (unsigned int)clahe_pixel(lut, g, ay, xs + 4 * k + j, tx_base, (w[k] >> (8 * j)) & 255u) << (8 * j);
        w[k] = o;
      }
      *reinterpret_cast<uint4*>(dst + xs) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
      for (int64_t x = xs; x < xe; ++x) dst[x] = clahe_pixel(lut, g, ay, x, tx_base, __ldg(src + x));
    }
  }
}

// ---- table path ----
// One CTA per (tile, section) of a batch of nb sections at `in` (H * W apart): histogram, clip, redistribute, scan, and the
// 256-byte LUT to luts[(section * tiles + tile) * 256].
__global__ void __launch_bounds__(kClaheThreads) clahe_lut_kernel(const uint8_t* __restrict__ in, int64_t nb, ClaheGeom g,
                                                                  uint8_t* __restrict__ luts) {
  __shared__ unsigned int sub[kClaheBins * 32];   // 32 lane-private sub-histograms, bin-major: lanes hit distinct banks
  __shared__ int64_t scan[2][kClaheBins];
  const int64_t tiles = g.tiles_x * g.tiles_y;
  const int lane = threadIdx.x & 31;
  const int64_t dr = blockDim.x / g.tw, dc = blockDim.x % g.tw;   // the step of a thread's (row, column) in the tile
  for (int64_t s = blockIdx.y; s < nb; s += gridDim.y)
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
      const uint8_t* sec = in + s * g.H * g.W;
      const int64_t ty = t / g.tiles_x, tx = t % g.tiles_x;
      __syncthreads();   // the previous tile is done with sub and scan
      for (int i = threadIdx.x; i < kClaheBins * 32; i += blockDim.x) sub[i] = 0;
      __syncthreads();
      unsigned int* mine = sub + lane;
      int64_t r = threadIdx.x / g.tw, c = threadIdx.x % g.tw;
      for (; r < g.th; r += dr, c += dc) {
        if (c >= g.tw) {
          c -= g.tw;
          if (++r >= g.th) break;
        }
        const uint8_t* row = sec + flt_fold(ty * g.th + r, g.H, kFltMirror) * g.W;
        atomicAdd(mine + ((unsigned int)__ldg(row + flt_fold(tx * g.tw + c, g.W, kFltMirror)) << 5), 1u);
      }
      __syncthreads();
      for (int b = threadIdx.x; b < kClaheBins; b += blockDim.x) {
        int64_t h = 0;
        for (int k = 0; k < 32; ++k) h += sub[b * 32 + ((k + b) & 31)];
        scan[0][b] = clahe_min(h, g.cl);
      }
      // inclusive scan of min(h, cl) over the bins (Hillis-Steele, ping-pong)
      int p = 0;
      for (int off = 1; off < kClaheBins; off <<= 1, p ^= 1) {
        __syncthreads();
        for (int b = threadIdx.x; b < kClaheBins; b += blockDim.x)
          scan[p ^ 1][b] = scan[p][b] + (b >= off ? scan[p][b - off] : 0);
      }
      __syncthreads();
      const ClaheSpread spread = clahe_spread(g.T - scan[p][kClaheBins - 1]);
      uint8_t* lut = luts + (s * tiles + t) * kClaheBins;
      for (int b = threadIdx.x; b < kClaheBins; b += blockDim.x) lut[b] = (uint8_t)clahe_lut_value(scan[p][b], b, spread, g.lut_scale);
    }
}

struct ClaheStagedLuts {
  const uint8_t* staged;   // 3 x 3 LUTs
  __device__ __forceinline__ int operator()(int64_t sy, int64_t sx, int v) const { return staged[(sy * 3 + sx) * kClaheBins + v]; }
};

// One CTA per (tile, section): the 3 x 3 LUTs around the tile (clamped at the grid's edges) into shared memory, then the
// tile's pixels of the section.
__global__ void __launch_bounds__(kClaheThreads) clahe_table_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                                    int64_t nb, ClaheGeom g, const uint8_t* __restrict__ luts) {
  __shared__ __align__(16) uint8_t staged[9 * kClaheBins];
  const int64_t tiles = g.tiles_x * g.tiles_y;
  for (int64_t s = blockIdx.y; s < nb; s += gridDim.y)
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int64_t ty = t / g.tiles_x, tx = t % g.tiles_x;
      const int64_t y0 = ty * g.th, x0 = tx * g.tw;
      if (y0 >= g.H || x0 >= g.W) continue;   // a tile of padding only (uniform across the CTA)
      __syncthreads();   // the previous tile is done with staged
      for (int i = threadIdx.x; i < 9 * kClaheBins; i += blockDim.x) {
        const int k = i / kClaheBins;
        const int64_t sy = clahe_min(clahe_max(ty - 1 + k / 3, 0), g.tiles_y - 1), sx = clahe_min(clahe_max(tx - 1 + k % 3, 0), g.tiles_x - 1);
        staged[i] = __ldg(luts + (s * tiles + sy * g.tiles_x + sx) * kClaheBins + i % kClaheBins);
      }
      __syncthreads();
      const int64_t off = s * g.H * g.W;
      clahe_write(in + off, out + off, g, y0, clahe_min(y0 + g.th, g.H), x0, clahe_min(x0 + g.tw, g.W), ty - 1, tx - 1,
                  ClaheStagedLuts{staged});
    }
}

// ---- small-tile path ----
// A CTA owns a region of ry x rx tiles and stages rs = (ry + 2) (rx + 2) tiles -- the region and the ring around it, clamped
// at the grid's edges -- as T keys each: the pixel's value where it counts towards sum_{i <= v} min(h[i], cl) (it is among the
// first cl pixels of its value in the tile, in raster order), 256 where it was clipped.  Then sum_{i <= v} min(h[i], cl) is
// the number of keys <= v.  Keys are pixel-major (key p of slot k at keys[p * slots + k]): neighbouring lanes read
// neighbouring tiles, so they hit neighbouring banks.
struct ClaheRegion {
  int64_t ry, rx;
};

inline int64_t clahe_small_smem_bytes(const ClaheGeom& g, const ClaheRegion& r) {
  const int64_t slots = (r.ry + 2) * (r.rx + 2);
  return slots * g.T * 3 + slots * (int64_t)sizeof(ClaheSpread);
}

// About 16 rows by 256 columns of pixels per CTA (16 groups of 16 bytes per row: one per thread), smaller while the staged
// tiles exceed kClaheSmallSmem.
inline ClaheRegion clahe_small_region(const ClaheGeom& g) {
  ClaheRegion r{clahe_min(g.tiles_y, clahe_max(1, 16 / g.th)), clahe_min(g.tiles_x, clahe_max(1, 256 / g.tw))};
  while (clahe_small_smem_bytes(g, r) > kClaheSmallSmem && (r.rx > 1 || r.ry > 1)) {
    if (r.rx >= r.ry) r.rx = (r.rx + 1) / 2;
    else r.ry = (r.ry + 1) / 2;
  }
  return r;
}

// lut(sy, sx, v) of staged slot (sy, sx) from its keys and its spread
struct ClaheKeyLuts {
  const uint16_t* keys;
  const ClaheSpread* spread;
  int T, cols, slots;
  float scale;
  __device__ __forceinline__ int operator()(int64_t sy, int64_t sx, int v) const {
    const int k = (int)sy * cols + (int)sx;
    int kept = 0;
    for (int p = 0; p < T; ++p) kept += keys[p * slots + k] <= v;
    return clahe_lut_value(kept, v, spread[k], scale);
  }
};

__global__ void __launch_bounds__(kClaheThreads) clahe_small_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                                    int64_t nz, ClaheGeom g, ClaheRegion reg) {
  extern __shared__ __align__(16) unsigned char clahe_smem[];
  const int64_t cols = reg.rx + 2, slots = (reg.ry + 2) * cols, T = g.T;
  ClaheSpread* spread = reinterpret_cast<ClaheSpread*>(clahe_smem);
  uint16_t* keys = reinterpret_cast<uint16_t*>(spread + slots);
  uint8_t* vals = reinterpret_cast<uint8_t*>(keys + slots * T);
  const int64_t regions_x = (g.tiles_x + reg.rx - 1) / reg.rx, regions = regions_x * ((g.tiles_y + reg.ry - 1) / reg.ry);
  for (int64_t s = blockIdx.y; s < nz; s += gridDim.y)
    for (int64_t q = blockIdx.x; q < regions; q += gridDim.x) {
      const int64_t ty0 = q / regions_x * reg.ry, tx0 = q % regions_x * reg.rx;
      const int64_t y0 = ty0 * g.th, x0 = tx0 * g.tw;
      if (y0 >= g.H || x0 >= g.W) continue;   // padding only (uniform across the CTA)
      const uint8_t* sec = in + s * g.H * g.W;
      __syncthreads();   // the previous region is done with the staged tiles
      for (int i = threadIdx.x; i < slots * T; i += blockDim.x) {   // slots * T is below 48 Ki (kClaheSmallSmem)
        const int k = i / (int)T, p = i % (int)T;
        const int64_t ty = clahe_min(clahe_max(ty0 - 1 + k / (int)cols, 0), g.tiles_y - 1);
        const int64_t tx = clahe_min(clahe_max(tx0 - 1 + k % (int)cols, 0), g.tiles_x - 1);
        const int64_t y = flt_fold(ty * g.th + p / (int)g.tw, g.H, kFltMirror), x = flt_fold(tx * g.tw + p % (int)g.tw, g.W, kFltMirror);
        vals[i] = __ldg(sec + y * g.W + x);
      }
      __syncthreads();
      for (int i = threadIdx.x; i < slots * T; i += blockDim.x) {
        const uint8_t v = vals[i];
        int64_t rank = 0;
        if (g.cl < T)
          for (int j = i - i % (int)T; j < i; ++j) rank += vals[j] == v;
        keys[(i % (int)T) * slots + i / (int)T] = rank < g.cl ? v : kClaheBins;
      }
      __syncthreads();
      for (int64_t k = threadIdx.x; k < slots; k += blockDim.x) {
        int64_t kept = 0;
        for (int64_t p = 0; p < T; ++p) kept += keys[p * slots + k] < kClaheBins;
        spread[k] = clahe_spread(T - kept);
      }
      __syncthreads();
      clahe_write(sec, out + s * g.H * g.W, g, y0, clahe_min(y0 + reg.ry * g.th, g.H), x0, clahe_min(x0 + reg.rx * g.tw, g.W),
                  ty0 - 1, tx0 - 1, ClaheKeyLuts{keys, spread, (int)T, (int)cols, (int)slots, g.lut_scale});
    }
}
