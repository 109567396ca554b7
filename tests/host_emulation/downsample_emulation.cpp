// TEST INFRASTRUCTURE: runs the device code of chunkflow_b200/csrc/downsample_kernels.cuh on the host, one "thread" in a
// grid of 1 x 1 x 1 (so every grid-stride loop walks the whole output), so that the kernels' LOGIC and the level plan are
// compared with oracle/downsample_oracle.py on machines without a GPU (tests/test_downsample_oracle.py builds this file with
// g++).  The launch geometry, 64-bit addressing at scale and unaligned device pointers are what the `-m gpu` tests add.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <vector>

#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
struct EmuDim { unsigned x = 0, y = 0, z = 0; };
static EmuDim blockIdx, threadIdx;
static struct { unsigned x = 1, y = 1, z = 1; } blockDim, gridDim;
struct uint4 { uint32_t x, y, z, w; };
struct uint2 { uint32_t x, y; };

#include "../../chunkflow_b200/csrc/downsample_kernels.cuh"

// uint8 averaging of (z,y,x) by (fz,fy,fx) into ceil(shape / factor), selected like cfb_downsample_average_device.
// -> 1 when the vectorised kernel ran, 0 for the generic one.
extern "C" int emu_average(const uint8_t* in, int64_t z, int64_t y, int64_t x, int64_t fz, int64_t fy, int64_t fx, uint8_t* out) {
  const DsDims s{z, y, x}, f{fz, fy, fx}, o{ds_ceil(z, fz), ds_ceil(y, fy), ds_ceil(x, fx)};
  if (!ds_average_vectorised(s, f, in, out)) {
    ds_average_kernel(in, s, o, f, out);
    return 0;
  }
  if (fz == 1) ds_average_x2_kernel<1, 2>(in, s, o, out);
  else ds_average_x2_kernel<2, 2>(in, s, o, out);
  return 1;
}

// The level plan: -> levels (-1 when refused); plan[5 i ..] = algorithm, preserved axis, output z, y, x of level i.
extern "C" int emu_plan(int kind, int64_t z, int64_t y, int64_t x, int64_t fz, int64_t fy, int64_t fx, int64_t* plan) {
  DsLevel levels[kDsMaxLevels];
  const char* why = "";
  const int n = ds_plan(kind, DsDims{z, y, x}, DsDims{fz, fy, fx}, levels, &why);
  for (int i = 0; i < n; ++i) {
    const int64_t row[5] = {levels[i].algo, levels[i].preserved, levels[i].out.z, levels[i].out.y, levels[i].out.x};
    std::memcpy(plan + 5 * i, row, sizeof(row));
  }
  return n;
}

template <typename T>
static void run_level(const DsLevel& l, int kind, const T* in, T* out) {
  if (l.algo == kDsStride) ds_stride_kernel<T>(in, l.in, l.out, l.factor, out);
  else if (l.algo == kDsCountless3d) ds_countless3d_kernel<T>(in, l.in, l.out, out);
  else if (kind == kDsU64) ds_countless2d_kernel<T, false>(in, l.in, l.out, l.preserved, out);
  else ds_countless2d_kernel<T, true>(in, l.in, l.out, l.preserved, out);
}

template <typename T>
static int run(int kind, const void* in, DsDims s, DsDims f, void* out) {
  DsLevel levels[kDsMaxLevels];
  const char* why = "";
  const int n = ds_plan(kind, s, f, levels, &why);
  if (n < 0) return n;
  if (n == 0) {
    std::memcpy(out, in, (size_t)(s.z * s.y * s.x) * sizeof(T));
    return 0;
  }
  std::vector<T> cur(static_cast<const T*>(in), static_cast<const T*>(in) + s.z * s.y * s.x), next;
  for (int i = 0; i < n; ++i) {
    const DsDims& o = levels[i].out;
    next.assign((size_t)(o.z * o.y * o.x), T(0));
    run_level<T>(levels[i], kind, cur.data(), next.data());
    cur.swap(next);
  }
  std::memcpy(out, cur.data(), cur.size() * sizeof(T));
  return n;
}

// kind: 0 bool (1 byte), 1 uint32, 2 uint64.  -> levels run, -1 when the factor is refused.
extern "C" int emu_segmentation(int kind, const void* in, int64_t z, int64_t y, int64_t x, int64_t fz, int64_t fy, int64_t fx,
                                void* out) {
  const DsDims s{z, y, x}, f{fz, fy, fx};
  if (kind == kDsBool) return run<uint8_t>(kind, in, s, f, out);
  if (kind == kDsU32) return run<uint32_t>(kind, in, s, f, out);
  return run<unsigned long long>(kind, in, s, f, out);
}
