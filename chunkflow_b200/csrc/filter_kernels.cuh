// Device code of `gaussian-filter` and the median filter (DESIGN.md section 0, row f8), included by filters.cu (which
// tests/host_emulation also compiles for the host, behind a one-lane CUDA shim).  The arithmetic is scipy.ndimage's, which
// the reference calls (chunk/base.py:846-853, plugins/gaussian_filter.py, plugins/median_filter.py), restated in
// oracle/filters_oracle.py:
//   gaussian  one 1-D pass per axis with the symmetric float64 weights w[0..r] (computed by the caller with numpy):
//             t = x[i] * w[0], then t = t + (x[i-j] + x[i+j]) * w[j] for j = r .. 1, every operation rounded on its own
//             (__dmul_rn / __dadd_rn: nvcc would contract a * b + c into an FMA), then a cast to the element type (uint8:
//             toward zero, float32: to nearest) that the next pass reads.  An axis without a pass has r = 0 and w = {1}:
//             x * 1 cast back is x, so it is the same as no pass.  Boundaries: reflect.
//   median    element V / 2 of the sorted window of V elements; the window of extent s spans offsets -(s/2) .. s-1-(s/2).
// flt_fold is the one index map per boundary mode, shared by both filters.  Every index is 64-bit.
//
// The gaussian works in place on the chunk, and a tile reads its neighbours' halos, so no CTA may overwrite input another
// still reads.  The library runs it on batches of whole sections through a workspace (filters.cu):
//   no channel pass  flt_gaussian_yx_kernel  chunk -> workspace, then a copy workspace -> chunk;
//   channel pass     flt_gaussian_c_kernel   chunk -> workspace, then flt_gaussian_yx_kernel workspace -> chunk.
// A section never reads another (there is no z-halo), so once a batch has been read into the workspace its sections of the
// chunk are free to be written.  Traffic per batch: one read and one write of the chunk, plus one write and one read of the
// workspace.  The workspace holds as many sections as fit kFltWorkspaceTarget (at least one), so that its write and read can
// be served by the 50 MB L2; whether they are was not measured, so count the HBM traffic as up to twice the chunk's.
// Every operand is converted to float64 where it is used, so a pass costs 2 r + 1 conversions per element on top of its
// 3 r + 1 operations.

#include "fold.cuh"

struct FltDims {
  int64_t n[4];   // (c, z, y, x); a 3-D chunk has c = 1
};

constexpr int kFltMaxRadius = 64;
constexpr int kFltMaxWindow = 125;
constexpr int64_t kFltWorkspaceTarget = 32ll << 20;

struct FltWeights {
  double w[kFltMaxRadius + 1];
  int r;
};

template <typename T>
__device__ __forceinline__ T flt_cast(double t);
template <>
__device__ __forceinline__ uint8_t flt_cast<uint8_t>(double t) { return (uint8_t)__double2uint_rz(t); }
template <>
__device__ __forceinline__ float flt_cast<float>(double t) { return __double2float_rn(t); }

// One output of a pass: x(k) reads the element at offset k from the centre (already folded by the caller's addressing).
template <typename T, typename Read>
__device__ __forceinline__ T flt_correlate(const FltWeights& w, Read x) {
  double t = __dmul_rn((double)x(0), w.w[0]);
  for (int j = w.r; j >= 1; --j) t = __dadd_rn(t, __dmul_rn(__dadd_rn((double)x(-j), (double)x(j)), w.w[j]));
  return flt_cast<T>(t);
}

// Plane (c, zb) of a batch: element (y, x) at base + c * cs + zb * zs + y * X + x.
struct FltPlanes {
  int64_t cs, zs;
};

// The y pass then the x pass of every (c, zb) plane of a batch (nc channels, nz sections), src -> dst (never the same
// memory).  A CTA owns a kFltTy x kFltTx output tile: it loads the tile plus its reflected halo into shared memory, runs the y
// pass over the tile's rows and the halo's columns into a second buffer, casting, and the x pass from there to dst.
constexpr int kFltTy = 32, kFltTx = 64, kFltThreads = 256;

inline int64_t flt_yx_smem_bytes(int ry, int rx, int64_t esize) {
  return (int64_t)(kFltTy + 2 * ry + kFltTy) * (kFltTx + 2 * rx) * esize;
}

template <typename T>
__global__ void __launch_bounds__(kFltThreads) flt_gaussian_yx_kernel(const T* __restrict__ src, FltPlanes sp, T* __restrict__ dst,
                                                                       FltPlanes dp, int64_t nc, int64_t nz, int64_t Y, int64_t X,
                                                                       FltWeights wy, FltWeights wx) {
  extern __shared__ __align__(16) unsigned char flt_smem[];
  const int ry = wy.r, rx = wx.r;
  const int ah = kFltTy + 2 * ry, aw = kFltTx + 2 * rx;
  T* a = reinterpret_cast<T*>(flt_smem);   // ah x aw: input tile with halo
  T* b = a + ah * aw;                      // kFltTy x aw: after the y pass
  const int64_t tiles_y = (Y + kFltTy - 1) / kFltTy, tiles_x = (X + kFltTx - 1) / kFltTx;
  for (int64_t p = blockIdx.z; p < nc * nz; p += gridDim.z) {
    const int64_t c = p / nz, zb = p % nz;
    const T* s = src + c * sp.cs + zb * sp.zs;
    T* d = dst + c * dp.cs + zb * dp.zs;
    for (int64_t ty = blockIdx.y; ty < tiles_y; ty += gridDim.y)
      for (int64_t tx = blockIdx.x; tx < tiles_x; tx += gridDim.x) {
        const int64_t y0 = ty * kFltTy, x0 = tx * kFltTx;
        __syncthreads();   // the previous tile's x pass has read b
        for (int k = threadIdx.x; k < ah * aw; k += blockDim.x) {
          const int ly = k / aw, lx = k % aw;
          const int64_t gy = flt_fold(y0 - ry + ly, Y, kFltReflect), gx = flt_fold(x0 - rx + lx, X, kFltReflect);
          a[k] = s[gy * X + gx];
        }
        __syncthreads();
        for (int k = threadIdx.x; k < kFltTy * aw; k += blockDim.x) {
          const int ly = k / aw, lx = k % aw;
          if (y0 + ly < Y) b[k] = flt_correlate<T>(wy, [&](int j) { return a[(ly + ry + j) * aw + lx]; });
        }
        __syncthreads();
        for (int k = threadIdx.x; k < kFltTy * kFltTx; k += blockDim.x) {
          const int ly = k / kFltTx, lx = k % kFltTx;
          if (y0 + ly < Y && x0 + lx < X)
            d[(y0 + ly) * X + x0 + lx] = flt_correlate<T>(wx, [&](int j) { return b[ly * aw + lx + rx + j]; });
        }
      }
  }
}

// The channel pass of a (c, z, y, x) chunk's sections (the reference filters the (c, y, x) block of every z): every element
// of nz sections, src -> dst, the channel axis reflected.  Blocks walk the (c, zb) planes in y and z, the (y, x) elements in x.
template <typename T>
__global__ void __launch_bounds__(kFltThreads) flt_gaussian_c_kernel(const T* __restrict__ src, FltPlanes sp, T* __restrict__ dst,
                                                                      FltPlanes dp, int64_t nc, int64_t nz, int64_t yx, FltWeights wc) {
  for (int64_t c = blockIdx.z; c < nc; c += gridDim.z)
    for (int64_t zb = blockIdx.y; zb < nz; zb += gridDim.y)
      for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < yx; e += (int64_t)gridDim.x * blockDim.x) {
        const T* s = src + zb * sp.zs + e;
        dst[c * dp.cs + zb * dp.zs + e] = flt_correlate<T>(wc, [&](int j) { return s[flt_fold(c + j, nc, kFltReflect) * sp.cs]; });
      }
}

// ---- median ----
template <typename T>
__device__ __forceinline__ T flt_top();
template <>
__device__ __forceinline__ uint8_t flt_top<uint8_t>() { return 0xFF; }
template <>
__device__ __forceinline__ float flt_top<float>() { return __int_as_float(0x7f800000); }   // +inf

template <typename T>
__device__ __forceinline__ void flt_order(T& a, T& b) {
  const T lo = a < b ? a : b, hi = a < b ? b : a;
  a = lo;
  b = hi;
}

// The flat index of window element k = (k0, k1, k2, k3) around pos, or -1 where the constant mode reads its 0.
__device__ __forceinline__ int64_t flt_window_at(const int64_t (&pos)[4], const int (&k)[4], const FltDims& n,
                                                 const FltDims& size, int mode) {
  int64_t at = 0;
  bool inside = true;
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const int64_t f = flt_fold(pos[d] + k[d] - size.n[d] / 2, n.n[d], mode);
    inside = inside && f >= 0;
    at = at * n.n[d] + (f < 0 ? 0 : f);
  }
  return inside ? at : -1;
}

__device__ __forceinline__ void flt_next(int (&k)[4], const FltDims& size) {
#pragma unroll
  for (int d = 3; d >= 0; --d) {
    if (++k[d] < size.n[d]) return;
    k[d] = 0;
  }
}

// Element V / 2 of the sorted window (V = volume elements, the extents in size; n = the array's (c, z, y, x) extents).
// kCap > 0: the window is gathered into registers and padded to kCap (a power of two) with the type's largest value -- pads
// sort behind every real element, so the first V sorted elements are the window's -- and a bitonic network sorts it.
// kCap == 0 (windows of more than 32 elements): the window goes to a local array and is sorted by insertion.
template <typename T, int kCap>
__global__ void __launch_bounds__(kFltThreads) flt_median_kernel(const T* __restrict__ in, FltDims n, FltDims size, int mode,
                                                                  T* __restrict__ out) {
  const int64_t total = n.n[0] * n.n[1] * n.n[2] * n.n[3];
  const int volume = (int)(size.n[0] * size.n[1] * size.n[2] * size.n[3]);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t pos[4], rest = i;
#pragma unroll
    for (int d = 3; d >= 0; --d) {
      pos[d] = rest % n.n[d];
      rest /= n.n[d];
    }
    int k[4] = {0, 0, 0, 0};
    if constexpr (kCap > 0) {
      T v[kCap];
#pragma unroll
      for (int e = 0; e < kCap; ++e) {
        v[e] = flt_top<T>();
        if (e < volume) {
          const int64_t at = flt_window_at(pos, k, n, size, mode);
          v[e] = at < 0 ? T(0) : in[at];
          flt_next(k, size);
        }
      }
#pragma unroll
      for (int s = 2; s <= kCap; s <<= 1)
#pragma unroll
        for (int j = s >> 1; j > 0; j >>= 1)
#pragma unroll
          for (int e = 0; e < kCap; ++e) {
            const int o = e ^ j;
            if (o > e) {
              if ((e & s) == 0) flt_order(v[e], v[o]);
              else flt_order(v[o], v[e]);
            }
          }
      T m = v[0];
#pragma unroll
      for (int e = 1; e < kCap; ++e)
        if (e == volume / 2) m = v[e];
      out[i] = m;
    } else {
      T v[kFltMaxWindow];
      for (int e = 0; e < volume; ++e) {
        const int64_t at = flt_window_at(pos, k, n, size, mode);
        T x = at < 0 ? T(0) : in[at];
        int j = e;
        for (; j > 0 && x < v[j - 1]; --j) v[j] = v[j - 1];
        v[j] = x;
        flt_next(k, size);
      }
      out[i] = v[volume / 2];
    }
  }
}

// size (3, 1, 1) along z of (c, z, y, x): a thread owns one (c, y, x) column and walks z keeping the 3-deep window, so the
// chunk is read once and written once.  Folded neighbours (z = 0 and z = Z - 1) are read where the mode puts them.
template <typename T>
__device__ __forceinline__ T flt_median3(T a, T b, T c) {
  const T lo = a < b ? a : b, hi = a < b ? b : a;
  const T m = hi < c ? hi : c;
  return lo < m ? m : lo;
}

template <typename T>
__global__ void __launch_bounds__(kFltThreads) flt_median_z3_kernel(const T* __restrict__ in, FltDims n, int mode,
                                                                     T* __restrict__ out) {
  const int64_t Z = n.n[1], yx = n.n[2] * n.n[3], columns = n.n[0] * yx;
  for (int64_t col = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; col < columns; col += (int64_t)gridDim.x * blockDim.x) {
    const T* s = in + (col / yx) * Z * yx + col % yx;
    T* d = out + (col / yx) * Z * yx + col % yx;
    auto at = [&](int64_t z) {
      const int64_t f = flt_fold(z, Z, mode);
      return f < 0 ? T(0) : s[f * yx];
    };
    T lo = at(-1), mid = s[0];
    for (int64_t z = 0; z < Z; ++z) {
      const T hi = z + 1 < Z ? s[(z + 1) * yx] : at(z + 1);
      d[z * yx] = flt_median3(lo, mid, hi);
      lo = mid;
      mid = hi;
    }
  }
}

// Which median kernel serves a window: -1 the z walk, else the kCap of flt_median_kernel.
inline int flt_median_path(const FltDims& size) {
  const int64_t v = size.n[0] * size.n[1] * size.n[2] * size.n[3];
  if (size.n[0] == 1 && size.n[1] == 3 && size.n[2] == 1 && size.n[3] == 1) return -1;
  return v <= 4 ? 4 : v <= 16 ? 16 : v <= 32 ? 32 : 0;
}
