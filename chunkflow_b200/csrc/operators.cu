// Operators either side of `inference`, on the device (SURVEY.md section 8 f3), so that a chunk can stay in HBM between
// operators instead of crossing PCIe (the 12.9 GB affinity map of a 1024^3 chunk):
//   upstream    normalize-contrast  reference chunk/image/base.py:30-132  (per-section histogram -> LUT -> apply, uint8)
//   both sides  maskout             reference chunk/base.py:811-829       (multiply by a coarser mask, integer factor)
//   downstream  crop-margin         reference chunk/base.py:691-726
//   downstream  quantize            reference chunk/affinity_map/base.py:33-57 (affinity -> uint8 image)
// All four are HBM-bound byte/float streams: 16-byte vector accesses, grid = a multiple of the SM count, no tensor cores.
// Results are bit-identical to the reference's numpy code (oracle/operators_oracle.py, tests/golden/operators.npz),
// including its quirks (normalize_contrast: the whole-array pass also runs after the per-section pass; 255-bin histograms).
#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

int sm_count_ops() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  return n;
}

// ------------------------------------------------------------------------------------------
// normalize-contrast
// ------------------------------------------------------------------------------------------
// Per-section 256-bin histogram.  grid = (blocks per section, Z).  32 lane-private sub-histograms interleaved so that
// counter (bin, lane) sits in bank `lane`: the shared-memory atomics of one warp instruction never conflict (a single
// shared table serialises ~3.5x on the birthday collisions of 32 lanes in 32 banks).  Algorithmic traffic: 1 B / voxel.
constexpr int kMlp = 4;  // independent 16-byte accesses per thread and loop trip of the streaming kernels below

__global__ void __launch_bounds__(256) section_hist_kernel(const uint8_t* __restrict__ img, int64_t section_elems,
                                                           unsigned long long* __restrict__ hist) {
  __shared__ unsigned int sh[256 * 32];
  for (int i = threadIdx.x; i < 256 * 32; i += 256) sh[i] = 0;
  __syncthreads();
  unsigned int* mine = sh + (threadIdx.x & 31);
  const uint8_t* sec = img + (int64_t)blockIdx.y * section_elems;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  // 16-byte body where the section start is 16-byte aligned, scalar head / tail otherwise
  const uintptr_t addr = reinterpret_cast<uintptr_t>(sec);
  const int64_t head_want = (int64_t)((16 - (addr & 15)) & 15);
  const int64_t head = section_elems < head_want ? section_elems : head_want;
  const int64_t nvec = (section_elems - head) / 16;
  const uint4* v = reinterpret_cast<const uint4*>(sec + head);
  auto count16 = [&](const uint4 q) {
    const unsigned int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      atomicAdd(mine + ((w[k] & 255u) << 5), 1u);
      atomicAdd(mine + (((w[k] >> 8) & 255u) << 5), 1u);
      atomicAdd(mine + (((w[k] >> 16) & 255u) << 5), 1u);
      atomicAdd(mine + ((w[k] >> 24) << 5), 1u);
    }
  };
  // the shared-memory atomics order the loop body, so the loads of later vectors cannot be hoisted by the compiler:
  // kMlp independent 16-byte loads are issued first (bytes in flight per SM, not the atomics, were the limit)
  int64_t i = tid;
  for (; i + (kMlp - 1) * stride < nvec; i += kMlp * stride) {
    uint4 q[kMlp];
#pragma unroll
    for (int k = 0; k < kMlp; ++k) q[k] = __ldg(v + i + k * stride);
#pragma unroll
    for (int k = 0; k < kMlp; ++k) count16(q[k]);
  }
  for (; i < nvec; i += stride) count16(__ldg(v + i));
  for (int64_t i = tid; i < head; i += stride) atomicAdd(mine + ((unsigned int)sec[i] << 5), 1u);
  for (int64_t i = head + nvec * 16 + tid; i < section_elems; i += stride) atomicAdd(mine + ((unsigned int)sec[i] << 5), 1u);
  __syncthreads();
  unsigned int c = 0;
#pragma unroll 8
  for (int j = 0; j < 32; ++j) c += sh[threadIdx.x * 32 + ((j + threadIdx.x) & 31)];  // rotated: conflict-free reads
  if (c) atomicAdd(&hist[(int64_t)blockIdx.y * 256 + threadIdx.x], (unsigned long long)c);
}

// Clamping values + lookup table of ONE histogram, exactly as the reference computes them (image/base.py:30-91):
// cdf without bin 0, over 255 bins unless the value 255 occurs (np.bincount minlength=255), double-precision
// fractions, float32 table arithmetic with separate (unfused) subtract / multiply, clip, round half to even.
// A block of 256 threads: thread 0 builds the prefix sums and finds both clamping values by binary search (the
// fraction cdf / total is monotone in the bin index, so "the last bin before the first one whose fraction exceeds
// the clip" -- the reference's two linear scans -- is a lower-bound search), then every thread writes one entry.
// `has` = false where the reference returns None (lower == upper, or an empty histogram): no transform.
struct LutScratch {
  unsigned long long cdf[256];
  int lower, upper, has;
};

__device__ __forceinline__ int first_fraction_above(const unsigned long long* cdf, int nbins, double total, double clip) {
  int lo = 0, hi = nbins;  // first i with cdf[i] / total > clip; nbins if there is none
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ddiv_rn((double)cdf[mid], total) > clip) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__device__ void build_lut_block(const unsigned long long* hist /* shared or global, 256 bins */, double lower_clip,
                                double upper_clip, int minval, int maxval, LutScratch& sc, uint8_t* lut /* 256 entries */) {
  if (threadIdx.x == 0) {
    const int nbins = hist[255] ? 256 : 255;
    unsigned long long acc = 0;
    sc.cdf[0] = 0;  // bin 0 (pure black) carries no information (image/base.py:38)
    for (int i = 1; i < nbins; ++i) { acc += hist[i]; sc.cdf[i] = acc; }
    int lower = 0, upper = 0;
    if (acc != 0) {
      const double total = (double)acc;
      int j = first_fraction_above(sc.cdf, nbins, total, lower_clip);
      lower = j < nbins ? (j > 0 ? j - 1 : 0) : nbins - 1;
      j = first_fraction_above(sc.cdf, nbins, total, 1.0 - upper_clip);
      upper = j < nbins ? (j > 0 ? j - 1 : 0) : nbins - 1;
    }
    sc.lower = lower; sc.upper = upper; sc.has = lower != upper;
  }
  __syncthreads();
  if (sc.has) {
    const float scale = __double2float_rn(__ddiv_rn((double)maxval, (double)sc.upper - (double)sc.lower));
    float t = __fmul_rn(__fsub_rn((float)threadIdx.x, (float)sc.lower), scale);
    t = fminf(fmaxf(t, (float)minval), (float)maxval);
    lut[threadIdx.x] = (uint8_t)(int)rintf(t);
  }
}

// One block per section: section table (identity where the reference applies none).
__global__ void __launch_bounds__(256) section_lut_kernel(const unsigned long long* __restrict__ hist, double lower_clip,
                                                          double upper_clip, int minval, int maxval, uint8_t* __restrict__ luts) {
  __shared__ unsigned long long h[256];
  __shared__ LutScratch sc;
  __shared__ uint8_t lut[256];
  h[threadIdx.x] = hist[(size_t)blockIdx.x * 256 + threadIdx.x];
  lut[threadIdx.x] = (uint8_t)threadIdx.x;
  __syncthreads();
  build_lut_block(h, lower_clip, upper_clip, minval, maxval, sc, lut);
  luts[(size_t)blockIdx.x * 256 + threadIdx.x] = lut[threadIdx.x];
}

// The reference's trailing whole-array pass (the for loop's else clause) sees the per-section RESULT.  Its histogram is
// the section histograms pushed through the section tables -- no second pass over the data ...
__global__ void __launch_bounds__(256) scatter_hist_kernel(const unsigned long long* __restrict__ hist,
                                                           const uint8_t* __restrict__ luts, unsigned long long* __restrict__ g) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  const unsigned long long c = hist[i];
  if (c) atomicAdd(&g[luts[i]], c);
}

// ... its table (glut[256], glut[256] = 1 when there is one) ...
__global__ void __launch_bounds__(256) global_lut_kernel(const unsigned long long* __restrict__ g, double lower_clip,
                                                         double upper_clip, int minval, int maxval, uint8_t* __restrict__ glut) {
  __shared__ unsigned long long h[256];
  __shared__ LutScratch sc;
  __shared__ uint8_t lut[256];
  h[threadIdx.x] = g[threadIdx.x];
  lut[threadIdx.x] = (uint8_t)threadIdx.x;
  __syncthreads();
  build_lut_block(h, lower_clip, upper_clip, minval, maxval, sc, lut);
  glut[threadIdx.x] = lut[threadIdx.x];
}

// ... is composed into every section table, so that ONE apply pass produces the final values.
__global__ void __launch_bounds__(256) compose_lut_kernel(const uint8_t* __restrict__ glut, uint8_t* __restrict__ luts) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  luts[i] = glut[luts[i]];
}

// out[i] = lut[section][img[i]] in place.  The table is replicated per lane (entry (value, lane) in bank `lane`), so
// the 16 lookups of a thread never conflict.  Algorithmic traffic: 1 B read + 1 B written per voxel.
__global__ void __launch_bounds__(256) apply_lut_kernel(uint8_t* __restrict__ img, int64_t section_elems,
                                                        const uint8_t* __restrict__ luts) {
  __shared__ unsigned int rep[256 * 32];
  {
    const unsigned int mine = luts[(size_t)blockIdx.y * 256 + threadIdx.x];
#pragma unroll 8
    for (int j = 0; j < 32; ++j) rep[threadIdx.x * 32 + ((j + threadIdx.x) & 31)] = mine;  // rotated: conflict-free writes
  }
  __syncthreads();
  const unsigned int* lut = rep + (threadIdx.x & 31);
  uint8_t* sec = img + (int64_t)blockIdx.y * section_elems;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(sec);
  const int64_t head_want = (int64_t)((16 - (addr & 15)) & 15);
  const int64_t head = section_elems < head_want ? section_elems : head_want;
  const int64_t nvec = (section_elems - head) / 16;
  uint4* v = reinterpret_cast<uint4*>(sec + head);
  auto map16 = [&](const uint4 q) {
    unsigned int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      w[k] = lut[(w[k] & 255u) << 5] | (lut[((w[k] >> 8) & 255u) << 5] << 8) | (lut[((w[k] >> 16) & 255u) << 5] << 16) |
             (lut[(w[k] >> 24) << 5] << 24);
    return make_uint4(w[0], w[1], w[2], w[3]);
  };
  int64_t i = tid;
  for (; i + (kMlp - 1) * stride < nvec; i += kMlp * stride) {   // kMlp loads in flight before the first store (in place: img is read and written)
    uint4 q[kMlp];
#pragma unroll
    for (int k = 0; k < kMlp; ++k) q[k] = v[i + k * stride];
#pragma unroll
    for (int k = 0; k < kMlp; ++k) v[i + k * stride] = map16(q[k]);
  }
  for (; i < nvec; i += stride) v[i] = map16(v[i]);
  for (int64_t i = tid; i < head; i += stride) sec[i] = (uint8_t)lut[(unsigned int)sec[i] << 5];
  for (int64_t i = head + nvec * 16 + tid; i < section_elems; i += stride) sec[i] = (uint8_t)lut[(unsigned int)sec[i] << 5];
}

// ------------------------------------------------------------------------------------------
// maskout: chunk[c, z, y, x] *= mask[z / fz, y / fy, x / fx]   (numpy in-place multiply, dtype of the chunk)
// ------------------------------------------------------------------------------------------
template <typename T, typename M>
__device__ __forceinline__ T mul_as(T v, M m);
template <> __device__ __forceinline__ uint8_t mul_as<uint8_t, uint8_t>(uint8_t v, uint8_t m) { return (uint8_t)(v * m); }
template <> __device__ __forceinline__ float mul_as<float, uint8_t>(float v, uint8_t m) { return __fmul_rn(v, (float)m); }
template <> __device__ __forceinline__ float mul_as<float, float>(float v, float m) { return __fmul_rn(v, m); }

// Rows are the unit (x is the fastest axis; grid = (row groups of a plane, channel-planes)): `tpr` threads (a power of
// two <= 256) cover one row with 16 bytes each, so a block works on 256 / tpr rows at a time -- narrow uint8 rows would
// otherwise leave most of the block idle.  No division per element: the mask index advances incrementally.
template <typename T, typename M>
__global__ void __launch_bounds__(256) maskout_kernel(T* __restrict__ chunk, int64_t rows, int Z, int Y, int X,
                                                      const M* __restrict__ mask, int MY, int MX, int fz, int fy, int fx,
                                                      int tpr) {
  constexpr int V = 16 / sizeof(T);
  const int64_t planes = rows / Y;  // channels * Z
  const int rpb = 256 / tpr, rsub = threadIdx.x / tpr, tx = threadIdx.x % tpr;
  const int ystep = gridDim.x * rpb;
  // rows whose pitch keeps every row start 16-byte aligned take the vector path with kMlp rows per thread and trip: all
  // their 16-byte loads are issued before the first multiply / store (in-place streams are bound by the bytes in flight)
  const bool rows_aligned = (reinterpret_cast<uintptr_t>(chunk) & 15) == 0 && ((int64_t)X * sizeof(T)) % 16 == 0;
  for (int64_t cz = blockIdx.y; cz < planes; cz += gridDim.y) {
    const int z = (int)(cz % Z);
    const M* mplane = mask + (int64_t)(z / fz) * MY * MX;
    for (int y0 = blockIdx.x * rpb + rsub; y0 < Y; y0 += kMlp * ystep) {
      if (rows_aligned) {
        for (int x0 = tx * V; x0 < X; x0 += tpr * V) {   // X % V == 0 here: every vector is whole
          uint4 pack[kMlp];
#pragma unroll
          for (int u = 0; u < kMlp; ++u)
            if (y0 + u * ystep < Y) pack[u] = *reinterpret_cast<const uint4*>(chunk + (cz * Y + y0 + u * ystep) * X + x0);
#pragma unroll
          for (int u = 0; u < kMlp; ++u) {
            const int y = y0 + u * ystep;
            if (y >= Y) continue;
            const M* mrow = mplane + (int64_t)(y / fy) * MX;
            int q = x0 / fx, r = x0 - q * fx;
            if constexpr (std::is_same<T, uint8_t>::value && std::is_same<M, uint8_t>::value) {
              if ((fx & 3) == 0) {
                // four voxels of a 32-bit word share one mask value: two 16-bit lanes per multiply, each byte modulo 256
                // (255 * 255 < 2^16: no carry between lanes) -- the per-byte path is bound by integer instructions
                uint32_t w[4];
                memcpy(w, &pack[u], 16);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  const uint32_t m = __ldg(mrow + q);
                  w[k] = (((w[k] & 0x00FF00FFu) * m) & 0x00FF00FFu) | ((((w[k] >> 8) & 0x00FF00FFu) * m & 0x00FF00FFu) << 8);
                  r += 4;
                  if (r == fx) { r = 0; ++q; }
                }
                memcpy(&pack[u], w, 16);
                *reinterpret_cast<uint4*>(chunk + (cz * Y + y) * X + x0) = pack[u];
                continue;
              }
            }
            T e[V];
            memcpy(e, &pack[u], 16);
            M m = __ldg(mrow + q);  // one mask load per run of fx voxels
#pragma unroll
            for (int k = 0; k < V; ++k) {
              e[k] = mul_as<T, M>(e[k], m);
              if (++r == fx) { r = 0; ++q; if (k + 1 < V) m = __ldg(mrow + q); }
            }
            memcpy(&pack[u], e, 16);
            *reinterpret_cast<uint4*>(chunk + (cz * Y + y) * X + x0) = pack[u];
          }
        }
      } else {
        for (int u = 0; u < kMlp; ++u) {
          const int y = y0 + u * ystep;
          if (y >= Y) break;
          T* prow = chunk + (cz * Y + y) * X;
          const M* mrow = mplane + (int64_t)(y / fy) * MX;
          for (int x0 = tx * V; x0 < X; x0 += tpr * V) {
            T* p = prow + x0;
            int q = x0 / fx, r = x0 - q * fx;
            for (int k = 0; k < V && x0 + k < X; ++k) {
              p[k] = mul_as<T, M>(p[k], __ldg(mrow + q));
              if (++r == fx) { r = 0; ++q; }
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// crop-margin: dst = src[..., lo_z : Z - hi_z, lo_y : Y - hi_y, lo_x : X - hi_x]  (dense copy of the sub-box)
// ------------------------------------------------------------------------------------------
// Rows are the unit, `tpr` threads per row as above; a row is OX * sizeof(T) contiguous bytes on both sides, copied with
// the widest access the alignment of this row pair allows (16 B, 4 B or single elements).
template <typename T>
__global__ void __launch_bounds__(256) crop_kernel(const T* __restrict__ src, int64_t channels, int Z, int Y, int X, int lz,
                                                   int ly, int lx, int OZ, int OY, int OX, T* __restrict__ dst, int tpr) {
  const int64_t planes = channels * OZ;
  const int row_bytes = OX * (int)sizeof(T);
  const int rpb = 256 / tpr, rsub = threadIdx.x / tpr, tx = threadIdx.x % tpr;
  for (int64_t cz = blockIdx.y; cz < planes; cz += gridDim.y)
  for (int y = blockIdx.x * rpb + rsub; y < OY; y += gridDim.x * rpb) {
    const int z = (int)(cz % OZ);
    const int64_t c = cz / OZ;
    const T* s = src + ((c * Z + (z + lz)) * Y + (y + ly)) * (int64_t)X + lx;
    T* d = dst + (cz * OY + y) * OX;
    const uintptr_t both = reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d) | (uintptr_t)row_bytes;
    if ((both & 15) == 0) {
      const uint4* s4 = reinterpret_cast<const uint4*>(s);
      uint4* d4 = reinterpret_cast<uint4*>(d);
      for (int i = tx; i < row_bytes / 16; i += tpr) d4[i] = __ldg(s4 + i);
    } else if ((both & 3) == 0) {
      const uint32_t* s1 = reinterpret_cast<const uint32_t*>(s);
      uint32_t* d1 = reinterpret_cast<uint32_t*>(d);
      for (int i = tx; i < row_bytes / 4; i += tpr) d1[i] = __ldg(s1 + i);
    } else {
      for (int i = tx; i < OX; i += tpr) d[i] = __ldg(s + i);
    }
  }
}

// ------------------------------------------------------------------------------------------
// quantize: uint8(((a0 + a1) / 2) * 255) ('xy') or uint8(a_last * 255) ('z'); float32 arithmetic, C truncation
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t to_u8(float v) { return (uint8_t)(int)v; }

__global__ void __launch_bounds__(256) quantize_kernel(const float* __restrict__ a0, const float* __restrict__ a1, int64_t n,
                                                       uint8_t* __restrict__ out) {
  const bool vec = ((reinterpret_cast<uintptr_t>(a0) | reinterpret_cast<uintptr_t>(a1)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 3) == 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x, tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nvec = vec ? n / 4 : 0;
  for (int64_t i = tid; i < nvec; i += stride) {
    const float4 p = __ldg(reinterpret_cast<const float4*>(a0) + i);
    float4 q = p;
    if (a1) {
      const float4 s = __ldg(reinterpret_cast<const float4*>(a1) + i);
      q.x = __fdiv_rn(__fadd_rn(p.x, s.x), 2.f); q.y = __fdiv_rn(__fadd_rn(p.y, s.y), 2.f);
      q.z = __fdiv_rn(__fadd_rn(p.z, s.z), 2.f); q.w = __fdiv_rn(__fadd_rn(p.w, s.w), 2.f);
    }
    uchar4 o;
    o.x = to_u8(__fmul_rn(q.x, 255.f)); o.y = to_u8(__fmul_rn(q.y, 255.f));
    o.z = to_u8(__fmul_rn(q.z, 255.f)); o.w = to_u8(__fmul_rn(q.w, 255.f));
    reinterpret_cast<uchar4*>(out)[i] = o;
  }
  for (int64_t i = nvec * 4 + tid; i < n; i += stride) {
    float v = a0[i];
    if (a1) v = __fdiv_rn(__fadd_rn(v, a1[i]), 2.f);
    out[i] = to_u8(__fmul_rn(v, 255.f));
  }
}

int grid_for(int64_t work_items, int threads = 256) {
  const int64_t want = ceil_div64(work_items, threads);
  const int64_t cap = (int64_t)sm_count_ops() * 8;  // 8 resident CTAs of 256 threads per SM
  return (int)std::max<int64_t>(1, std::min<int64_t>(want, cap));
}

int threads_per_row(int64_t row_bytes) {  // smallest power of two >= ceil(row_bytes / 16), at most 256
  int t = 1;
  while (t < 256 && (int64_t)t * 16 < row_bytes) t <<= 1;
  return t;
}

dim3 grid_rows(int64_t planes, int64_t rows_per_plane, int tpr) {  // row kernels: about 16 CTAs of 256 threads per SM
  const int64_t gy = std::min<int64_t>(planes, 65535);
  const int64_t groups = ceil_div64(rows_per_plane, 256 / tpr);
  const int64_t gx = std::max<int64_t>(1, std::min<int64_t>(groups, ceil_div64((int64_t)sm_count_ops() * 16, gy)));
  return dim3((unsigned)gx, (unsigned)gy);
}

void check_dims(int64_t c, int64_t z, int64_t y, int64_t x) {
  if (c < 1 || z < 1 || y < 1 || x < 1 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX)
    throw std::invalid_argument("chunk dimensions must be positive and each spatial axis below 2^31");
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" {

int cfb_normalize_contrast_device(void* d_image, int64_t z, int64_t y, int64_t x, double lower_clip_fraction,
                                  double upper_clip_fraction, int32_t minval, int32_t maxval, int32_t per_section,
                                  void* stream) {
  return guarded([&]() -> int {
    check_dims(1, z, y, x);
    if (!d_image) throw std::invalid_argument("normalize_contrast: null image");
    if (minval < 0 || maxval > 255 || minval > maxval) throw std::invalid_argument("normalize_contrast: need 0 <= minval <= maxval <= 255");
    // reference image/base.py:113: with per_section=False NOTHING runs (the whole-array branch belongs to the for loop)
    if (!per_section) return CFB_OK;
    if (z > 65535) throw std::invalid_argument("normalize_contrast: at most 65535 sections per call");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int64_t section = y * x;
    unsigned long long* hist = nullptr;  // (z + 1) x 256: section histograms, then the whole-array histogram
    uint8_t* luts = nullptr;             // (z + 1) x 256: section tables, then the whole-array table
    CFB_CUDA(cudaMallocAsync(&hist, (size_t)(z + 1) * 256 * sizeof(unsigned long long), s));
    CFB_CUDA(cudaMallocAsync(&luts, (size_t)(z + 1) * 256, s));
    CFB_CUDA(cudaMemsetAsync(hist, 0, (size_t)(z + 1) * 256 * sizeof(unsigned long long), s));
    unsigned long long* ghist = hist + (size_t)z * 256;
    uint8_t* glut = luts + (size_t)z * 256;
    const int per_sec = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(section, 256 * 64), ceil_div64((int64_t)sm_count_ops() * 6, z)));
    const dim3 grid(per_sec, (unsigned)z);
    section_hist_kernel<<<grid, 256, 0, s>>>(static_cast<const uint8_t*>(d_image), section, hist);
    CFB_LAUNCH_CHECK();
    section_lut_kernel<<<(unsigned)z, 256, 0, s>>>(hist, lower_clip_fraction, upper_clip_fraction, minval, maxval, luts);
    CFB_LAUNCH_CHECK();
    scatter_hist_kernel<<<(unsigned)z, 256, 0, s>>>(hist, luts, ghist);
    CFB_LAUNCH_CHECK();
    global_lut_kernel<<<1, 256, 0, s>>>(ghist, lower_clip_fraction, upper_clip_fraction, minval, maxval, glut);
    CFB_LAUNCH_CHECK();
    compose_lut_kernel<<<(unsigned)z, 256, 0, s>>>(glut, luts);
    CFB_LAUNCH_CHECK();
    apply_lut_kernel<<<grid, 256, 0, s>>>(static_cast<uint8_t*>(d_image), section, luts);
    CFB_LAUNCH_CHECK();
    CFB_CUDA(cudaFreeAsync(hist, s));
    CFB_CUDA(cudaFreeAsync(luts, s));
    return CFB_OK;
  });
}

int cfb_maskout_device(void* d_chunk, int32_t chunk_dtype, int64_t channels, int64_t z, int64_t y, int64_t x,
                       const void* d_mask, int32_t mask_dtype, int64_t fz, int64_t fy, int64_t fx, void* stream) {
  return guarded([&]() -> int {
    check_dims(channels, z, y, x);
    if (!d_chunk || !d_mask) throw std::invalid_argument("maskout: null pointer");
    if (fz < 1 || fy < 1 || fx < 1 || z % fz || y % fy || x % fx)
      throw std::invalid_argument("maskout: the chunk size must be the mask size times the integer voxel-size factor");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int64_t rows = channels * z * y;
    const int MY = (int)(y / fy), MX = (int)(x / fx);
    const int tpr = threads_per_row(x * (chunk_dtype == CFB_DTYPE_U8 ? 1 : 4));
    if (chunk_dtype == CFB_DTYPE_U8 && mask_dtype == CFB_DTYPE_U8) {
      maskout_kernel<uint8_t, uint8_t><<<grid_rows(channels * z, y, tpr), 256, 0, s>>>(
          static_cast<uint8_t*>(d_chunk), rows, (int)z, (int)y, (int)x, static_cast<const uint8_t*>(d_mask), MY, MX, (int)fz, (int)fy, (int)fx, tpr);
    } else if (chunk_dtype == CFB_DTYPE_F32 && mask_dtype == CFB_DTYPE_U8) {
      maskout_kernel<float, uint8_t><<<grid_rows(channels * z, y, tpr), 256, 0, s>>>(
          static_cast<float*>(d_chunk), rows, (int)z, (int)y, (int)x, static_cast<const uint8_t*>(d_mask), MY, MX, (int)fz, (int)fy, (int)fx, tpr);
    } else if (chunk_dtype == CFB_DTYPE_F32 && mask_dtype == CFB_DTYPE_F32) {
      maskout_kernel<float, float><<<grid_rows(channels * z, y, tpr), 256, 0, s>>>(
          static_cast<float*>(d_chunk), rows, (int)z, (int)y, (int)x, static_cast<const float*>(d_mask), MY, MX, (int)fz, (int)fy, (int)fx, tpr);
    } else {
      // numpy refuses uint8 *= float32 (casting rule 'same_kind'), and so do we
      throw std::invalid_argument("maskout: unsupported dtype pair (chunk uint8 needs a uint8/bool mask)");
    }
    CFB_LAUNCH_CHECK();
    return CFB_OK;
  });
}

int cfb_crop_margin_device(const void* d_src, int32_t dtype, int64_t channels, int64_t z, int64_t y, int64_t x,
                           const int64_t margin[6], void* d_dst, void* stream) {
  return guarded([&]() -> int {
    check_dims(channels, z, y, x);
    if (!d_src || !d_dst || !margin) throw std::invalid_argument("crop_margin: null pointer");
    for (int i = 0; i < 6; ++i)
      if (margin[i] < 0) throw std::invalid_argument("crop_margin: negative margin");
    const int64_t oz = z - margin[0] - margin[3], oy = y - margin[1] - margin[4], ox = x - margin[2] - margin[5];
    if (oz < 1 || oy < 1 || ox < 1) throw std::invalid_argument("crop_margin: the margins leave nothing");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int tpr = threads_per_row(ox * (dtype == CFB_DTYPE_U8 ? 1 : 4));
    if (dtype == CFB_DTYPE_U8) {
      crop_kernel<uint8_t><<<grid_rows(channels * oz, oy, tpr), 256, 0, s>>>(static_cast<const uint8_t*>(d_src), channels, (int)z, (int)y, (int)x,
                                                          (int)margin[0], (int)margin[1], (int)margin[2], (int)oz, (int)oy, (int)ox,
                                                          static_cast<uint8_t*>(d_dst), tpr);
    } else if (dtype == CFB_DTYPE_F32) {
      crop_kernel<float><<<grid_rows(channels * oz, oy, tpr), 256, 0, s>>>(static_cast<const float*>(d_src), channels, (int)z, (int)y, (int)x,
                                                        (int)margin[0], (int)margin[1], (int)margin[2], (int)oz, (int)oy, (int)ox,
                                                        static_cast<float*>(d_dst), tpr);
    } else {
      throw std::invalid_argument("crop_margin: dtype must be CFB_DTYPE_U8 or CFB_DTYPE_F32");
    }
    CFB_LAUNCH_CHECK();
    return CFB_OK;
  });
}

int cfb_quantize_device(const float* d_affinity, int64_t channels, int64_t z, int64_t y, int64_t x, int32_t mode,
                        uint8_t* d_out, void* stream) {
  return guarded([&]() -> int {
    check_dims(channels, z, y, x);
    if (!d_affinity || !d_out) throw std::invalid_argument("quantize: null pointer");
    const int64_t n = z * y * x;
    const float *a0, *a1;
    if (mode == CFB_QUANTIZE_XY) {
      if (channels < 2) throw std::invalid_argument("quantize: mode xy needs at least two channels");
      a0 = d_affinity; a1 = d_affinity + n;
    } else if (mode == CFB_QUANTIZE_Z) {
      a0 = d_affinity + (channels - 1) * n; a1 = nullptr;
    } else {
      throw std::invalid_argument("quantize: only support xy and z mode");  // reference affinity_map/base.py:51
    }
    quantize_kernel<<<grid_for(ceil_div64(n, 4)), 256, 0, static_cast<cudaStream_t>(stream)>>>(a0, a1, n, d_out);
    CFB_LAUNCH_CHECK();
    return CFB_OK;
  });
}

}  // extern "C"
