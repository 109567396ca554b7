// TEST INFRASTRUCTURE: runs the device code of chunkflow_b200/csrc/clahe_kernels.cuh on the host, one "thread" in a grid of
// 1 x 1 x 1 (so every grid-stride loop walks all the work), so that the kernels' LOGIC -- tiles read through the reflected
// index map, the LUT scan, the closed form of the small-tile path, the staged neighbour slots, batches of sections, the
// 16-byte groups -- is compared with oracle/clahe_oracle.py on machines without a GPU (tests/test_clahe_oracle.py builds this
// file with g++ -ffp-contract=off, so that a * b + c is not fused, as __fmul_rn / __fadd_rn guarantee on the device).
#include <cfenv>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __shared__
#define __align__(n) __attribute__((aligned(n)))
#define __launch_bounds__(...)
struct EmuDim { unsigned x = 0, y = 0, z = 0; };
static EmuDim blockIdx, threadIdx;
static struct { unsigned x = 1, y = 1, z = 1; } blockDim, gridDim;
struct uint4 { unsigned int x, y, z, w; };
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return uint4{a, b, c, d}; }
static inline void __syncthreads() {}
static inline unsigned atomicAdd(unsigned* p, unsigned v) { const unsigned old = *p; *p += v; return old; }
static inline uint8_t __ldg(const uint8_t* p) { return *p; }
static inline uint4 __ldg(const uint4* p) { return *p; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline int __float2int_rn(float a) { return (int)std::nearbyint(a); }   // the default rounding mode: half to even
alignas(16) unsigned char clahe_smem[1 << 24];

#include "../../chunkflow_b200/csrc/clahe_kernels.cuh"

// The launch sequence of clahe.cu's clahe_run with the path forced (-1: chosen from T as the library does, 0 table, 1 small
// tile) and table batches of `batch` sections.  -> the path taken.
extern "C" int emu_clahe(const uint8_t* in, uint8_t* out, int64_t z, int64_t y, int64_t x, double clip, int64_t tiles_x,
                         int64_t tiles_y, int path, int64_t batch) {
  std::fesetround(FE_TONEAREST);
  const ClaheGeom g = clahe_geometry(y, x, tiles_x, tiles_y, clip);
  if (path < 0) path = clahe_small_tiles(g) ? 1 : 0;
  if (path == 1) {
    clahe_small_kernel(in, out, z, g, clahe_small_region(g));
    return 1;
  }
  std::vector<uint8_t> luts((size_t)(batch * g.tiles_x * g.tiles_y * kClaheBins));
  for (int64_t z0 = 0; z0 < z; z0 += batch) {
    const int64_t nb = z - z0 < batch ? z - z0 : batch;
    clahe_lut_kernel(in + z0 * y * x, nb, g, luts.data());
    clahe_table_kernel(in + z0 * y * x, out + z0 * y * x, nb, g, luts.data());
  }
  return 0;
}

// The region of tiles one CTA of the small-tile path owns, and the tile size: (ry, rx, th, tw).
extern "C" void emu_small_region(int64_t y, int64_t x, int64_t tiles_x, int64_t tiles_y, int64_t* out) {
  const ClaheGeom g = clahe_geometry(y, x, tiles_x, tiles_y, 0.0);
  const ClaheRegion r = clahe_small_region(g);
  out[0] = r.ry;
  out[1] = r.rx;
  out[2] = g.th;
  out[3] = g.tw;
}
