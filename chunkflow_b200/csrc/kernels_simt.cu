// fp32 CUDA-core network kernels (sm_90a).  See kernels_simt.cuh.
#include "kernels_simt.cuh"

namespace cfb {
namespace {

// ---- 3x3x3 convolution -------------------------------------------------------------
// Block = 256 threads = 16 (x groups of 4 voxels) x 16 (rows); output tile 1 x 16 x 64,
// 16 output channels per block.  Per input channel the 3 x 18 x 66 halo tile and the
// 16 x 27 weights are staged in shared memory; every thread keeps 16 x 4 accumulators.
constexpr int kTX = 64, kTY = 16, kCO = 16;
constexpr int kPitch = 68;  // floats; 66 used, 16-byte aligned rows

__global__ void __launch_bounds__(256)
conv3_f32_kernel(const float* __restrict__ in0, int c0, const float* __restrict__ in1, int c1,
                 const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out,
                 int cout, Int3 sz, int tiles_x, int relu) {
  __shared__ __align__(16) float s_in[3][kTY + 2][kPitch];
  __shared__ __align__(16) float s_w[9][kCO][4];

  const int cin = c0 + c1;
  const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
  const int z = blockIdx.y;
  const int co_tiles = cout / kCO;
  const int b = blockIdx.z / co_tiles, co_base = (blockIdx.z % co_tiles) * kCO;
  const int x0 = tile_x * kTX, y0 = tile_y * kTY;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t plane = (int64_t)sz.y * sz.x, volume = plane * sz.z;

  float acc[kCO][4];
#pragma unroll
  for (int c = 0; c < kCO; ++c) acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f;

  for (int ci = 0; ci < cin; ++ci) {
    const float* src = ci < c0 ? in0 + ((int64_t)b * c0 + ci) * volume
                               : in1 + ((int64_t)b * c1 + (ci - c0)) * volume;
    __syncthreads();  // previous iteration done with s_in / s_w
    for (int i = threadIdx.x; i < 3 * (kTY + 2) * (kTX + 2); i += 256) {
      int c = i % (kTX + 2);
      int r = (i / (kTX + 2)) % (kTY + 2);
      int d = i / ((kTX + 2) * (kTY + 2));
      int gz = z + d - 1, gy = y0 + r - 1, gx = x0 + c - 1;
      float v = 0.f;
      if (gz >= 0 && gz < sz.z && gy >= 0 && gy < sz.y && gx >= 0 && gx < sz.x)
        v = __ldg(src + (int64_t)gz * plane + (int64_t)gy * sz.x + gx);
      s_in[d][r][c] = v;
    }
    for (int i = threadIdx.x; i < kCO * 27; i += 256) {
      int co = i / 27, tap = i % 27;
      s_w[tap / 3][co][tap % 3] = __ldg(w + ((int64_t)(co_base + co) * cin + ci) * 27 + tap);
    }
    __syncthreads();
#pragma unroll
    for (int dz = 0; dz < 3; ++dz) {
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const float* row = &s_in[dz][ty + dy][tx * 4];
        const float4 a = *reinterpret_cast<const float4*>(row);
        const float2 bq = *reinterpret_cast<const float2*>(row + 4);
        const float v[6] = {a.x, a.y, a.z, a.w, bq.x, bq.y};
#pragma unroll
        for (int co = 0; co < kCO; ++co) {
          const float4 wv = *reinterpret_cast<const float4*>(&s_w[dz * 3 + dy][co][0]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            acc[co][k] = fmaf(wv.x, v[k], acc[co][k]);
            acc[co][k] = fmaf(wv.y, v[k + 1], acc[co][k]);
            acc[co][k] = fmaf(wv.z, v[k + 2], acc[co][k]);
          }
        }
      }
    }
  }

  const int y = y0 + ty, x = x0 + tx * 4;
  if (y >= sz.y || x >= sz.x) return;
#pragma unroll
  for (int co = 0; co < kCO; ++co) {
    const float bv = bias ? __ldg(bias + co_base + co) : 0.f;
    float r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      r[k] = acc[co][k] + bv;
      if (relu) r[k] = r[k] < 0.f ? 0.f : r[k];  // NaN passes, like torch.relu
    }
    float* dst = out + ((int64_t)b * cout + co_base + co) * volume + (int64_t)z * plane + (int64_t)y * sz.x + x;
    if (x + 4 <= sz.x && (sz.x & 3) == 0) {
      *reinterpret_cast<float4*>(dst) = make_float4(r[0], r[1], r[2], r[3]);
    } else {
      for (int k = 0; k < 4 && x + k < sz.x; ++k) dst[k] = r[k];
    }
  }
}

__global__ void __launch_bounds__(256)
maxpool_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t planes, int Y, int X) {
  const int oy = Y / 2, ox = X / 2;
  const int64_t total = planes * oy * ox;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)(i % ox);
    int64_t r = i / ox;
    int y = (int)(r % oy);
    int64_t p = r / oy;
    const float* s = in + (p * Y + 2 * y) * X + 2 * x;
    const float2 a = *reinterpret_cast<const float2*>(s);
    const float2 c = *reinterpret_cast<const float2*>(s + X);
    out[i] = fmaxf(fmaxf(a.x, a.y), fmaxf(c.x, c.y));
  }
}

// One thread = one OUTPUT voxel, all output channels (<= 32).
template <int COUT>
__global__ void __launch_bounds__(256)
convT_f32_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                 float* __restrict__ out, int cin, int nb, Int3 isz) {
  extern __shared__ float s_wt[];  // [cin][4][COUT]  (tap = a*2+b)
  for (int i = threadIdx.x; i < cin * COUT * 4; i += blockDim.x) {
    int tap = i % 4, co = (i / 4) % COUT, ci = i / (4 * COUT);  // global layout (cin, cout, 1, 2, 2)
    s_wt[(ci * 4 + tap) * COUT + co] = w[i];
  }
  __syncthreads();
  const int OY = isz.y * 2, OX = isz.x * 2;
  const int64_t ovol = (int64_t)isz.z * OY * OX, ivol = (int64_t)isz.z * isz.y * isz.x;
  const int64_t total = (int64_t)nb * ovol;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)(i % OX);
    int64_t r = i / OX;
    int y = (int)(r % OY);
    r /= OY;
    int z = (int)(r % isz.z);
    int b = (int)(r / isz.z);
    const int tap = (y & 1) * 2 + (x & 1);
    const float* src = in + (int64_t)b * cin * ivol + ((int64_t)z * isz.y + (y >> 1)) * isz.x + (x >> 1);
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
    for (int ci = 0; ci < cin; ++ci) {
      const float v = __ldg(src + (int64_t)ci * ivol);
      const float* wp = &s_wt[(ci * 4 + tap) * COUT];
#pragma unroll
      for (int co = 0; co < COUT; ++co) acc[co] = fmaf(v, wp[co], acc[co]);
    }
    float* dst = out + (int64_t)b * COUT * ovol + ((int64_t)z * OY + y) * OX + x;
#pragma unroll
    for (int co = 0; co < COUT; ++co) dst[(int64_t)co * ovol] = acc[co] + __ldg(bias + co);
  }
}

__global__ void __launch_bounds__(256)
head_sigmoid_f32_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                        float* __restrict__ out, int cin, int cout, int nb, int64_t volume) {
  extern __shared__ float s_hw[];  // [cout][cin] + [cout]
  for (int i = threadIdx.x; i < cout * cin; i += blockDim.x) s_hw[i] = w[i];
  for (int i = threadIdx.x; i < cout; i += blockDim.x) s_hw[cout * cin + i] = bias[i];
  __syncthreads();
  const int64_t total = (int64_t)nb * volume;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i % volume, b = i / volume;
    const float* src = in + b * cin * volume + v;
    float acc[8];
    for (int co = 0; co < cout; ++co) acc[co] = s_hw[cout * cin + co];
    for (int ci = 0; ci < cin; ++ci) {
      const float a = __ldg(src + (int64_t)ci * volume);
      for (int co = 0; co < cout; ++co) acc[co] = fmaf(a, s_hw[co * cin + ci], acc[co]);
    }
    for (int co = 0; co < cout; ++co)
      out[(b * cout + co) * volume + v] = __fdiv_rn(1.0f, 1.0f + expf(-acc[co]));
  }
}

int grid_for(int64_t items) {
  int64_t b = ceil_div64(items, 256);
  if (b < 1) b = 1;
  if (b > 132 * 16) b = 132 * 16;
  return (int)b;
}

}  // namespace

void launch_conv3_f32(const float* in0, int c0, const float* in1, int c1, const float* w, const float* bias,
                      float* out, int cout, int nb, Int3 sz, bool relu, cudaStream_t s) {
  if (cout % kCO != 0) throw std::runtime_error("conv3_f32: cout must be a multiple of 16");
  const int tiles_x = ceil_div(sz.x, kTX), tiles_y = ceil_div(sz.y, kTY);
  dim3 grid(tiles_x * tiles_y, sz.z, nb * (cout / kCO));
  conv3_f32_kernel<<<grid, 256, 0, s>>>(in0, c0, in1, c1, w, bias, out, cout, sz, tiles_x, relu ? 1 : 0);
  CFB_LAUNCH_CHECK();
}

void launch_maxpool_f32(const float* in, float* out, int channels, int nb, Int3 isz, cudaStream_t s) {
  const int64_t planes = (int64_t)nb * channels * isz.z;
  maxpool_f32_kernel<<<grid_for(planes * (isz.y / 2) * (isz.x / 2)), 256, 0, s>>>(in, out, planes, isz.y, isz.x);
  CFB_LAUNCH_CHECK();
}

void launch_convT_f32(const float* in, const float* w, const float* bias, float* out, int cin, int cout, int nb,
                      Int3 isz, cudaStream_t s) {
  const int64_t items = (int64_t)nb * isz.z * isz.y * 2 * isz.x * 2;
  const size_t smem = (size_t)cin * cout * 4 * sizeof(float);
  if (cout == 32) {
    convT_f32_kernel<32><<<grid_for(items), 256, smem, s>>>(in, w, bias, out, cin, nb, isz);
  } else if (cout == 16) {
    convT_f32_kernel<16><<<grid_for(items), 256, smem, s>>>(in, w, bias, out, cin, nb, isz);
  } else {
    throw std::runtime_error("convT_f32: unsupported cout");
  }
  CFB_LAUNCH_CHECK();
}

void launch_head_sigmoid_f32(const float* in, const float* w, const float* bias, float* out, int cin, int cout,
                             int nb, Int3 sz, cudaStream_t s) {
  if (cout > 8) throw std::runtime_error("head: at most 8 output channels");
  const size_t smem = (size_t)(cout * cin + cout) * sizeof(float);
  head_sigmoid_f32_kernel<<<grid_for((int64_t)nb * vol(sz)), 256, smem, s>>>(in, w, bias, out, cin, cout, nb, vol(sz));
  CFB_LAUNCH_CHECK();
}

}  // namespace cfb
