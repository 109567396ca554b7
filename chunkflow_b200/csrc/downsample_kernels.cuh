// Device code of `downsample` (DESIGN.md section 0, row f7), included by downsample.cu (which tests/host_emulation also
// compiles for the host, behind a one-lane CUDA shim).  The arithmetic is the reference's vendored numpy downsampler (reference
// lib/igneous/downsample.py), restated in oracle/downsample_oracle.py:
//   average     uint8, any factor: floor(block sum / voxels in the block), the block clipped at the far edges;
//   countless2d one preserved axis: the other two halved, an odd side first grown by a copy of its first plane in front
//               (odd_to_even2d), so that output j reads inputs (max(2j - odd, 0), 2j + 1 - odd); with a, b, c, d the
//               (lower, lower), (lower, upper), (upper, lower), (upper, upper) voxels of the pair: a if a == b or a == c,
//               else b if b == c, else d;
//   countless3d 2x2x2 on even shapes: the 8 voxels in (z, y, x) ndindex order, i = 4 dz + 2 dy + dx.  A value seen >= 4
//               times wins, then >= 3 times, then >= 2 times among voxels 0..6; else voxel 7.  Between values of one rank
//               the one seen first wins (the reference's combinations are walked in lexicographic order, and two values
//               never share a position, so the first r-tuple of a value is decided by its first position);
//   stride      out[z, y, x] = in[z fz, y fy, x fx].
// The reference adds 1 to every id and takes 0 as "no pick".  Where it does so in the stored width, the all-ones id (the
// maximum of an unsigned type, -1 of a signed one) is never picked: countless3d always, countless2d for 64-bit ids
// (it widens 8-, 16- and 32-bit ones first).  kEveryIdCounts says which case a kernel is.
// Every kernel walks its output with a 3-D grid-stride loop (x threads, y and z blocks), 64-bit indices, no division.

struct DsDims {
  int64_t z, y, x;
};

#define DS_FOR_EACH_OUTPUT(o)                                                                         \
  for (int64_t oz = blockIdx.z; oz < (o).z; oz += gridDim.z)                                          \
    for (int64_t oy = blockIdx.y; oy < (o).y; oy += gridDim.y)                                        \
      for (int64_t ox = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; ox < (o).x;                   \
           ox += (int64_t)gridDim.x * blockDim.x)

// uint8 averaging.  The caller guarantees fz * fy * fx <= kDsMaxAverageBlock, so the sum fits 24 bits: where the reference's
// float32 sum is exact, and floor(sum / count) is what its float64 division and cast to uint8 give.
constexpr int64_t kDsMaxAverageBlock = 65793;   // 65793 * 255 < 2^24

__global__ void __launch_bounds__(256) ds_average_kernel(const uint8_t* __restrict__ in, DsDims s, DsDims o, DsDims f,
                                                          uint8_t* __restrict__ out) {
  DS_FOR_EACH_OUTPUT(o) {
    const int64_t z0 = oz * f.z, y0 = oy * f.y, x0 = ox * f.x;
    const int64_t z1 = z0 + f.z < s.z ? z0 + f.z : s.z;
    const int64_t y1 = y0 + f.y < s.y ? y0 + f.y : s.y;
    const int64_t x1 = x0 + f.x < s.x ? x0 + f.x : s.x;
    const int nz = (int)(z1 - z0), ny = (int)(y1 - y0), nx = (int)(x1 - x0);
    const uint8_t* plane = in + (z0 * s.y + y0) * s.x + x0;
    uint32_t sum = 0;
    for (int dz = 0; dz < nz; ++dz, plane += s.y * s.x) {
      const uint8_t* row = plane;
      for (int dy = 0; dy < ny; ++dy, row += s.x)
        for (int dx = 0; dx < nx; ++dx) sum += row[dx];
    }
    out[(oz * o.y + oy) * o.x + ox] = (uint8_t)(sum / (uint32_t)(nz * ny * nx));
  }
}

// uint8 averaging by (kFz, kFy, 2) -- the factors of an image pyramid (1,2,2) and a volume pyramid (2,2,2) -- on rows that are
// 16-byte aligned: a thread averages 8 outputs from one 16-byte load per input row, all kFz * kFy loads issued before the first
// add.  Each 32-bit word holds the two byte-pair sums of 4 input bytes in its 16-bit halves (at most 4 rows * 510 < 2^16).
// Rows past the far z / y edge are not loaded and not counted; x is never clipped (the row length is a multiple of 16).
template <int kFz, int kFy>
__global__ void __launch_bounds__(256) ds_average_x2_kernel(const uint8_t* __restrict__ in, DsDims s, DsDims o,
                                                             uint8_t* __restrict__ out) {
  constexpr int kRows = kFz * kFy;
  const DsDims groups = {o.z, o.y, o.x / 8};
  DS_FOR_EACH_OUTPUT(groups) {
    uint4 v[kRows];
    int rows = 0;
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
      const int64_t z = oz * kFz + r / kFy, y = oy * kFy + r % kFy;
      const bool inside = z < s.z && y < s.y;
      v[r] = inside ? *reinterpret_cast<const uint4*>(in + (z * s.y + y) * s.x + 16 * ox) : uint4{0, 0, 0, 0};
      rows += inside ? 1 : 0;
    }
    uint32_t pairs[4] = {0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
      const uint32_t w[4] = {v[r].x, v[r].y, v[r].z, v[r].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) pairs[k] += (w[k] & 0x00FF00FFu) + ((w[k] >> 8) & 0x00FF00FFu);
    }
    const uint32_t count = 2u * (uint32_t)rows;
    uint32_t packed[2] = {0, 0};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t sum = (pairs[j >> 1] >> (16 * (j & 1))) & 0xFFFFu;
      packed[j >> 2] |= (sum / count) << (8 * (j & 3));
    }
    *reinterpret_cast<uint2*>(out + (oz * o.y + oy) * o.x + 8 * ox) = uint2{packed[0], packed[1]};
  }
}

// The vectorised path serves (1,2,2) and (2,2,2) on rows of a multiple of 16 bytes starting at 16-byte aligned addresses
// (input) and 8-byte aligned ones (output); every other case takes ds_average_kernel.
inline bool ds_average_vectorised(DsDims s, DsDims f, const void* in, const void* out) {
  return f.x == 2 && f.y == 2 && (f.z == 1 || f.z == 2) && s.x % 16 == 0 && (uintptr_t)in % 16 == 0 && (uintptr_t)out % 8 == 0;
}

template <typename T>
__device__ __forceinline__ bool ds_counts(T v, bool every_id_counts) {
  return every_id_counts || v != (T)~(T)0;
}

template <typename T, bool kEveryIdCounts>
__device__ __forceinline__ T ds_countless2(T a, T b, T c, T d) {
  if (ds_counts(a, kEveryIdCounts) && (a == b || a == c)) return a;
  if (ds_counts(b, kEveryIdCounts) && b == c) return b;
  return d;
}

// The two inputs of output j along a halved axis of input extent n (odd n: the prepended copy of plane 0).
__device__ __forceinline__ void ds_pair(int64_t j, int64_t n, int64_t& i0, int64_t& i1) {
  const int64_t odd = n & 1;
  i0 = 2 * j - odd < 0 ? 0 : 2 * j - odd;
  i1 = 2 * j + 1 - odd;
}

// preserved: the axis (0 z, 1 y, 2 x) that keeps its extent.
template <typename T, bool kEveryIdCounts>
__global__ void __launch_bounds__(256) ds_countless2d_kernel(const T* __restrict__ in, DsDims s, DsDims o, int preserved,
                                                              T* __restrict__ out) {
  DS_FOR_EACH_OUTPUT(o) {
    int64_t z0 = oz, z1 = oz, y0 = oy, y1 = oy, x0 = ox, x1 = ox;
    if (preserved != 0) ds_pair(oz, s.z, z0, z1);
    if (preserved != 1) ds_pair(oy, s.y, y0, y1);
    if (preserved != 2) ds_pair(ox, s.x, x0, x1);
    // the two halved axes in (z, y, x) order are (u, v); b and c are interchangeable in the rule
    int64_t ia, ib, ic, id;
    if (preserved == 0) {
      ia = (z0 * s.y + y0) * s.x + x0; ib = (z0 * s.y + y0) * s.x + x1;
      ic = (z0 * s.y + y1) * s.x + x0; id = (z0 * s.y + y1) * s.x + x1;
    } else if (preserved == 1) {
      ia = (z0 * s.y + y0) * s.x + x0; ib = (z0 * s.y + y0) * s.x + x1;
      ic = (z1 * s.y + y0) * s.x + x0; id = (z1 * s.y + y0) * s.x + x1;
    } else {
      ia = (z0 * s.y + y0) * s.x + x0; ib = (z0 * s.y + y1) * s.x + x0;
      ic = (z1 * s.y + y0) * s.x + x0; id = (z1 * s.y + y1) * s.x + x0;
    }
    out[(oz * o.y + oy) * o.x + ox] = ds_countless2<T, kEveryIdCounts>(in[ia], in[ib], in[ic], in[id]);
  }
}

// The mode of a 2x2x2 block by ranks (see the top of this file); v[i] with i = 4 dz + 2 dy + dx.
template <typename T>
__device__ __forceinline__ T ds_countless8(const T (&v)[8]) {
  int count[8], count7[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    count[i] = 0;
    count7[i] = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = v[i] == v[j] ? 1 : 0;
      count[i] += e;
      if (j < 7) count7[i] += e;
    }
    if (!ds_counts(v[i], false)) count[i] = count7[i] = 0;
  }
#pragma unroll
  for (int r = 4; r >= 3; --r)
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (count[i] >= r) return v[i];
#pragma unroll
  for (int i = 0; i < 7; ++i)
    if (count7[i] >= 2) return v[i];
  return v[7];
}

template <typename T>
__global__ void __launch_bounds__(256) ds_countless3d_kernel(const T* __restrict__ in, DsDims s, DsDims o, T* __restrict__ out) {
  DS_FOR_EACH_OUTPUT(o) {
    T v[8];
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
        const T* row = in + ((2 * oz + dz) * s.y + 2 * oy + dy) * s.x + 2 * ox;
        v[4 * dz + 2 * dy] = row[0];
        v[4 * dz + 2 * dy + 1] = row[1];
      }
    out[(oz * o.y + oy) * o.x + ox] = ds_countless8(v);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) ds_stride_kernel(const T* __restrict__ in, DsDims s, DsDims o, DsDims f, T* __restrict__ out) {
  DS_FOR_EACH_OUTPUT(o) {
    out[(oz * o.y + oy) * o.x + ox] = in[(oz * f.z * s.y + oy * f.y) * s.x + ox * f.x];
  }
}

// ---- the level plan of downsample_segmentation (host code) ----
// The reference recurses: a 2x2x2 or 2x2 step, then the rest of the factor (factor // 2 here; the reference's factor / 2
// raises on every second level).  Each level is decided from the element kind, the level's shape and the remaining factor.
enum DsAlgo { kDsStride = 0, kDsCountless2d = 1, kDsCountless3d = 2 };
enum DsKind { kDsBool = 0, kDsU32 = 1, kDsU64 = 2 };
constexpr int kDsMaxLevels = 64;
constexpr int64_t kDsMaxFactorProduct = INT32_MAX;

struct DsLevel {
  int algo;
  int preserved;   // countless2d
  DsDims in, out, factor;   // factor: stride
};

inline bool ds_pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

inline int64_t ds_ceil(int64_t a, int64_t b) { return (a + b - 1) / b; }

// -> number of levels (0: the input is the result), or -1 with *why set when the factor is refused.
inline int ds_plan(int kind, DsDims shape, DsDims factor, DsLevel* levels, const char** why) {
  int n = 0;
  DsDims s = shape, f = factor;
  if (f.z <= 0 || f.y <= 0 || f.x <= 0) { *why = "downsample: factors below one make no sense"; return -1; }
  if (f.z > kDsMaxFactorProduct / f.y || f.z * f.y > kDsMaxFactorProduct / f.x) {
    *why = "downsample: the factor's product exceeds 2^31 - 1"; return -1;
  }
  for (;;) {
    if (f.z <= 0 || f.y <= 0 || f.x <= 0) {
      *why = "downsample: the factor's recursion leaves a factor of 0 on an axis with factor 1 (the reference raises)";
      return -1;
    }
    if (f.z == 1 && f.y == 1 && f.x == 1) return n;
    if (n == kDsMaxLevels) { *why = "downsample: too many levels"; return -1; }
    DsLevel& l = levels[n++];
    l.in = s;
    l.factor = f;
    l.preserved = -1;
    const bool pot = ds_pow2(f.z) && ds_pow2(f.y) && ds_pow2(f.x);   // the product is a power of two
    const bool has_one = f.z == 1 || f.y == 1 || f.x == 1;
    if (kind != kDsBool && pot && !has_one && !(s.z & 1) && !(s.y & 1) && !(s.x & 1)) {
      l.algo = kDsCountless3d;
      s = {s.z / 2, s.y / 2, s.x / 2};
      f = {f.z / 2, f.y / 2, f.x / 2};
      l.out = s;
      continue;
    }
    if (kind == kDsBool || !(pot && has_one)) {
      l.algo = kDsStride;
      l.out = {ds_ceil(s.z, f.z), ds_ceil(s.y, f.y), ds_ceil(s.x, f.x)};
      return n;
    }
    l.algo = kDsCountless2d;
    l.preserved = f.z == 1 ? 0 : f.y == 1 ? 1 : 2;
    s = {l.preserved == 0 ? s.z : (s.z + 1) / 2, l.preserved == 1 ? s.y : (s.y + 1) / 2, l.preserved == 2 ? s.x : (s.x + 1) / 2};
    f = {l.preserved == 0 ? 1 : f.z / 2, l.preserved == 1 ? 1 : f.y / 2, l.preserved == 2 ? 1 : f.x / 2};
    l.out = s;
  }
}
