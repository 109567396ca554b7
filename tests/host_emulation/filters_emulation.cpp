// TEST INFRASTRUCTURE: runs the device code of chunkflow_b200/csrc/filter_kernels.cuh on the host, one "thread" in a grid of
// 1 x 1 x 1 (so every grid-stride loop walks all the work), so that the kernels' LOGIC -- tiles, halos, batches of sections,
// the median paths -- is compared with oracle/filters_oracle.py on machines without a GPU (tests/test_filters_oracle.py builds
// this file with g++ -ffp-contract=off, so that a * b + c is not fused, as __dmul_rn / __dadd_rn guarantee on the device).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __shared__
#define __align__(n)
#define __launch_bounds__(...)
struct EmuDim { unsigned x = 0, y = 0, z = 0; };
static EmuDim blockIdx, threadIdx;
static struct { unsigned x = 1, y = 1, z = 1; } blockDim, gridDim;
static inline void __syncthreads() {}
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline unsigned __double2uint_rz(double t) { return (unsigned)t; }
static inline float __double2float_rn(double t) { return (float)t; }
static inline float __int_as_float(int v) { float f; std::memcpy(&f, &v, sizeof f); return f; }
alignas(16) unsigned char flt_smem[1 << 20];

#include "../../chunkflow_b200/csrc/filter_kernels.cuh"

static FltWeights weights(const double* w, int r) {
  FltWeights out{};
  out.w[0] = 1.0;
  if (w) std::memcpy(out.w, w, sizeof(double) * (r + 1));
  out.r = w ? r : 0;
  return out;
}

// The batch loop of filters.cu's flt_gaussian with batches of `batch` sections.
template <typename T>
static void gaussian(T* data, FltDims d, const double* wc, int rc, const double* wy, int ry, const double* wx, int rx, int64_t batch) {
  const int64_t C = d.n[0], Z = d.n[1], Y = d.n[2], X = d.n[3], yx = Y * X;
  std::vector<T> work((size_t)(batch * C * yx));
  const FltWeights c = weights(wc, rc), y = weights(wy, ry), x = weights(wx, rx);
  for (int64_t z0 = 0; z0 < Z; z0 += batch) {
    const int64_t nb = std::min(batch, Z - z0);
    const FltPlanes chunk{Z * yx, yx}, ws{nb * yx, yx};
    T* at = data + z0 * yx;
    if (wc) {
      flt_gaussian_c_kernel<T>(at, chunk, work.data(), ws, C, nb, yx, c);
      flt_gaussian_yx_kernel<T>(work.data(), ws, at, chunk, C, nb, Y, X, y, x);
    } else {
      flt_gaussian_yx_kernel<T>(at, chunk, work.data(), ws, C, nb, Y, X, y, x);
      for (int64_t k = 0; k < C; ++k) std::memcpy(at + k * Z * yx, work.data() + k * nb * yx, (size_t)(nb * yx) * sizeof(T));
    }
  }
}

// dtype 0 uint8, 1 float32; data (c, z, y, x) filtered in place.
extern "C" void emu_gaussian(int dtype, void* data, int64_t c, int64_t z, int64_t y, int64_t x, const double* wc, int rc,
                             const double* wy, int ry, const double* wx, int rx, int64_t batch) {
  const FltDims d{{c, z, y, x}};
  if (dtype == 0) gaussian<uint8_t>((uint8_t*)data, d, wc, rc, wy, ry, wx, rx, batch);
  else gaussian<float>((float*)data, d, wc, rc, wy, ry, wx, rx, batch);
}

template <typename T>
static int median(const T* in, FltDims n, FltDims s, int mode, T* out) {
  const int path = flt_median_path(s);
  if (path < 0) flt_median_z3_kernel<T>(in, n, mode, out);
  else if (path == 4) flt_median_kernel<T, 4>(in, n, s, mode, out);
  else if (path == 16) flt_median_kernel<T, 16>(in, n, s, mode, out);
  else if (path == 32) flt_median_kernel<T, 32>(in, n, s, mode, out);
  else flt_median_kernel<T, 0>(in, n, s, mode, out);
  return path;
}

// -> the path taken (-1 the z walk, else the register capacity, 0 the local-array kernel).
extern "C" int emu_median(int dtype, const void* in, int64_t c, int64_t z, int64_t y, int64_t x, const int64_t* size, int mode,
                          void* out) {
  const FltDims n{{c, z, y, x}}, s{{size[0], size[1], size[2], size[3]}};
  if (dtype == 0) return median<uint8_t>((const uint8_t*)in, n, s, mode, (uint8_t*)out);
  return median<float>((const float*)in, n, s, mode, (float*)out);
}
