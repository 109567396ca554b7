// CUDA-core kernels on the CP8 (chunk-planar fp16, optional hi/lo split) activation layout:
// layout conversion, the first (Cin = 1) convolution fused with patch extraction, max pooling,
// transposed convolution and the 1x1x1 head.  See kernels_conv.cuh.
#include "kernels_conv.cuh"

#include "act_format.cuh"
#include "chunkflow_b200.h"

namespace cfb {
namespace {

constexpr int kT = 256;

__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack2(uint32_t u) { return __half22float2(*reinterpret_cast<__half2*>(&u)); }

// 8 fp32 values -> hi record (and lo record = residual) of one voxel
__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  float h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) h[i] = __half2float(__float2half_rn(v[i]));
  hi = make_uint4(pack2(h[0], h[1]), pack2(h[2], h[3]), pack2(h[4], h[5]), pack2(h[6], h[7]));
  lo = make_uint4(pack2(v[0] - h[0], v[1] - h[1]), pack2(v[2] - h[2], v[3] - h[3]), pack2(v[4] - h[4], v[5] - h[5]),
                  pack2(v[6] - h[6], v[7] - h[7]));
}
__device__ __forceinline__ void unpack8(const uint4& r, float (&v)[8]) {
  float2 a = unpack2(r.x), b = unpack2(r.y), c = unpack2(r.z), d = unpack2(r.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
// Every kernel below takes the activation number format `fmt` (ActFmt: 1 = fp16, 2 = fp16 hi + lo, 3 = f16f8, see
// act_format.cuh) and addresses an 8-channel chunk by the index of its first plane, chunk * fmt_planes(fmt).
// load the 8 channels of the chunk whose first plane is `plane0` at voxel `vox` as fp32
__device__ __forceinline__ void load8(const uint4* __restrict__ base, size_t plane0, int fmt, size_t pvol, size_t vox,
                                      float (&v)[8]) {
  if (fmt == kFmtF16F8) {
    // H record of this chunk + its half of the L8 record of the K step (plane (chunk | 1, part 1))
    const uint4 h = __ldg(base + plane0 * pvol + vox);
    const uint2 l = __ldg(reinterpret_cast<const uint2*>(base + ((plane0 | 2) + 1) * pvol + vox) + ((plane0 >> 1) & 1));
    af_decode8(h, l.x, l.y, v);
    return;
  }
  unpack8(__ldg(base + plane0 * pvol + vox), v);
  if (fmt == kFmtF16x2) {
    float l[8];
    unpack8(__ldg(base + (plane0 + 1) * pvol + vox), l);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] += l[i];
  }
}
__device__ __forceinline__ void store8(uint4* __restrict__ base, size_t plane0, int fmt, size_t pvol, size_t vox,
                                       const float (&v)[8]) {
  if (fmt == kFmtF16F8) {
    float s[8], l[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i] = fminf(fmaxf(v[i] * kActAlpha, -kHalfMax), kHalfMax);
      const float h = __half2float(__float2half_rn(s[i]));
      l[i] = (s[i] - h) * kActLambda;
      s[i] = h;
    }
    base[plane0 * pvol + vox] = make_uint4(pack2(s[0], s[1]), pack2(s[2], s[3]), pack2(s[4], s[5]), pack2(s[6], s[7]));
    const int half = (int)((plane0 >> 1) & 1);  // which 8 of the 16 channels of the K step
    reinterpret_cast<uint2*>(base + ((plane0 & ~(size_t)2) + 1) * pvol + vox)[half] =
        make_uint2(af_pack_e4m3x4(v[0] * kActGamma, v[1] * kActGamma, v[2] * kActGamma, v[3] * kActGamma),
                   af_pack_e4m3x4(v[4] * kActGamma, v[5] * kActGamma, v[6] * kActGamma, v[7] * kActGamma));
    reinterpret_cast<uint2*>(base + ((plane0 | 2) + 1) * pvol + vox)[half] =
        make_uint2(af_pack_e4m3x4(l[0], l[1], l[2], l[3]), af_pack_e4m3x4(l[4], l[5], l[6], l[7]));
    return;
  }
  uint4 hi, lo;
  split8(v, hi, lo);
  base[plane0 * pvol + vox] = hi;
  if (fmt == kFmtF16x2) base[(plane0 + 1) * pvol + vox] = lo;
}

__global__ void __launch_bounds__(kT)
planar_to_cp8_kernel(const float* __restrict__ in, uint4* __restrict__ out, int channels, int parts, int nb, size_t pvol) {
  const int chunks = channels / 8;
  const size_t total = (size_t)nb * chunks * pvol;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t vox = i % pvol;
    const size_t bc = i / pvol;  // b * chunks + chunk
    const size_t b = bc / chunks, chunk = bc % chunks;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = in[((b * channels) + chunk * 8 + e) * pvol + vox];
    store8(out, bc * fmt_planes(parts), parts, pvol, vox, v);
  }
}

__global__ void __launch_bounds__(kT)
cp8_to_planar_kernel(const uint4* __restrict__ in, float* __restrict__ out, int channels, int parts, int nb, size_t pvol) {
  const int chunks = channels / 8;
  const size_t total = (size_t)nb * chunks * pvol;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t vox = i % pvol;
    const size_t bc = i / pvol;
    const size_t b = bc / chunks, chunk = bc % chunks;
    float v[8];
    load8(in, bc * fmt_planes(parts), parts, pvol, vox, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) out[((b * channels) + chunk * 8 + e) * pvol + vox] = v[e];
  }
}

// ---- first layer: extract + normalise + conv 1->16 + ReLU ---------------------------------
// SRC: 0 = uint8 chunk, 1 = float chunk, 2 = float patches (nb,1,Z,Y,X)
constexpr int kFX = 32, kFY = 8;
template <int SRC>
__global__ void __launch_bounds__(kT)
first_conv_cp8_kernel(const void* __restrict__ src, Int3 cs, const PatchPos* __restrict__ patches, Int3 ps,
                      const float* __restrict__ w, const float* __restrict__ bias, uint4* __restrict__ out, int parts,
                      int tiles_x) {
  __shared__ float s_in[3][kFY + 2][kFX + 2];
  __shared__ __align__(16) float s_w[27][16];
  __shared__ float s_b[16];
  const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
  const int z = blockIdx.y, b = blockIdx.z;
  const int x0 = tile_x * kFX, y0 = tile_y * kFY;
  int oz = 0, oy = 0, ox = 0, flags = 0;
  if (SRC != 2) { const PatchPos pp = patches[b]; oz = pp.iz; oy = pp.iy; ox = pp.ix; flags = pp.flags; }
  for (int i = threadIdx.x; i < 3 * (kFY + 2) * (kFX + 2); i += kT) {
    const int c = i % (kFX + 2), r = (i / (kFX + 2)) % (kFY + 2), d = i / ((kFX + 2) * (kFY + 2));
    const int gz = z + d - 1, gy = y0 + r - 1, gx = x0 + c - 1;
    float v = 0.f;  // zero padding at the PATCH border
    if (gz >= 0 && gz < ps.z && gy >= 0 && gy < ps.y && gx >= 0 && gx < ps.x) {
      int sy = gy, sx = gx;
      if (SRC != 2 && flags) tta_map(flags, ps.y, ps.x, gy, gx, sy, sx);  // augmented variant reads the original patch
      if (SRC == 0) {
        v = __fdiv_rn((float)static_cast<const uint8_t*>(src)[((size_t)(oz + gz) * cs.y + (oy + sy)) * cs.x + ox + sx], 255.0f);
      } else if (SRC == 1) {
        v = static_cast<const float*>(src)[((size_t)(oz + gz) * cs.y + (oy + sy)) * cs.x + ox + sx];
      } else {
        v = static_cast<const float*>(src)[(((size_t)b * ps.z + gz) * ps.y + gy) * ps.x + gx];
      }
    }
    s_in[d][r][c] = v;
  }
  for (int i = threadIdx.x; i < 27 * 16; i += kT) s_w[i / 16][i % 16] = w[(i % 16) * 27 + (i / 16)];
  if (threadIdx.x < 16) s_b[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int lx = threadIdx.x % kFX, ly = threadIdx.x / kFX;
  const int x = x0 + lx, y = y0 + ly;
  if (x >= ps.x || y >= ps.y) return;
  float acc[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) acc[c] = 0.f;
#pragma unroll
  for (int t = 0; t < 27; ++t) {
    const float v = s_in[t / 9][ly + (t / 3) % 3][lx + t % 3];
    const float4* wp = reinterpret_cast<const float4*>(&s_w[t][0]);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 wv = wp[q];
      acc[q * 4 + 0] = fmaf(wv.x, v, acc[q * 4 + 0]);
      acc[q * 4 + 1] = fmaf(wv.y, v, acc[q * 4 + 1]);
      acc[q * 4 + 2] = fmaf(wv.z, v, acc[q * 4 + 2]);
      acc[q * 4 + 3] = fmaf(wv.w, v, acc[q * 4 + 3]);
    }
  }
  const size_t pvol = (size_t)ps.z * ps.y * ps.x;
  const size_t vox = ((size_t)z * ps.y + y) * ps.x + x;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float t = acc[h * 8 + i] + s_b[h * 8 + i]; v[i] = t < 0.f ? 0.f : t; }  // NaN passes, like torch.relu
    store8(out, ((size_t)b * 2 + h) * fmt_planes(parts), parts, pvol, vox, v);
  }
}

// Same layer with the weights as constant-bank operands (FirstConvW kernel parameter): identical FMA order and results.
template <int SRC>
__global__ void __launch_bounds__(kT)
first_conv_cp8_const_kernel(const void* __restrict__ src, Int3 cs, const PatchPos* __restrict__ patches, Int3 ps,
                            const __grid_constant__ FirstConvW W, uint4* __restrict__ out, int parts, int tiles_x) {
  __shared__ float s_in[3][kFY + 2][kFX + 2];
  const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
  const int z = blockIdx.y, b = blockIdx.z;
  const int x0 = tile_x * kFX, y0 = tile_y * kFY;
  const PatchPos pp = patches[b];
  const int oz = pp.iz, oy = pp.iy, ox = pp.ix, flags = pp.flags;
  for (int i = threadIdx.x; i < 3 * (kFY + 2) * (kFX + 2); i += kT) {
    const int c = i % (kFX + 2), r = (i / (kFX + 2)) % (kFY + 2), d = i / ((kFX + 2) * (kFY + 2));
    const int gz = z + d - 1, gy = y0 + r - 1, gx = x0 + c - 1;
    float v = 0.f;  // zero padding at the PATCH border
    if (gz >= 0 && gz < ps.z && gy >= 0 && gy < ps.y && gx >= 0 && gx < ps.x) {
      int sy = gy, sx = gx;
      if (flags) tta_map(flags, ps.y, ps.x, gy, gx, sy, sx);  // augmented variant reads the original patch
      const size_t idx = ((size_t)(oz + gz) * cs.y + (oy + sy)) * cs.x + ox + sx;
      v = SRC == 0 ? __fdiv_rn((float)static_cast<const uint8_t*>(src)[idx], 255.0f) : static_cast<const float*>(src)[idx];
    }
    s_in[d][r][c] = v;
  }
  __syncthreads();
  const int lx = threadIdx.x % kFX, ly = threadIdx.x / kFX;
  const int x = x0 + lx, y = y0 + ly;
  if (x >= ps.x || y >= ps.y) return;
  float acc[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) acc[c] = 0.f;
#pragma unroll
  for (int t = 0; t < 27; ++t) {
    const float v = s_in[t / 9][ly + (t / 3) % 3][lx + t % 3];
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[c] = fmaf(W.w[t][c], v, acc[c]);
  }
  const size_t pvol = (size_t)ps.z * ps.y * ps.x;
  const size_t vox = ((size_t)z * ps.y + y) * ps.x + x;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float t = acc[h * 8 + i] + W.b[h * 8 + i]; v[i] = t < 0.f ? 0.f : t; }  // NaN passes, like torch.relu
    store8(out, ((size_t)b * 2 + h) * fmt_planes(parts), parts, pvol, vox, v);
  }
}

// ---- max pool (1,2,2) ---------------------------------------------------------------------
__global__ void __launch_bounds__(kT)
maxpool_cp8_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int parts, size_t nplanes_chunks, Int3 isz) {
  const int OY = isz.y / 2, OX = isz.x / 2;
  const size_t ipvol = (size_t)isz.z * isz.y * isz.x, opvol = (size_t)isz.z * OY * OX;
  const size_t total = nplanes_chunks * opvol;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t ov = i % opvol, bc = i / opvol;
    const int x = (int)(ov % OX), y = (int)((ov / OX) % OY), z = (int)(ov / ((size_t)OX * OY));
    float m[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = -INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const size_t iv = ((size_t)z * isz.y + 2 * y + (k >> 1)) * isz.x + 2 * x + (k & 1);
      float v[8];
      load8(in, bc * fmt_planes(parts), parts, ipvol, iv, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) m[e] = fmaxf(m[e], v[e]);
    }
    store8(out, bc * fmt_planes(parts), parts, opvol, ov, m);
  }
}

// ---- transposed convolution kernel = stride = (1,2,2), one thread per OUTPUT voxel --------
template <int COUT>
__global__ void __launch_bounds__(kT)
convT_cp8_kernel(const uint4* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                 uint4* __restrict__ out, int cin, int parts, int nb, Int3 isz) {
  extern __shared__ float s_wt[];  // [cin][4][COUT]
  for (int i = threadIdx.x; i < cin * COUT * 4; i += blockDim.x) {
    const int tap = i % 4, co = (i / 4) % COUT, ci = i / (4 * COUT);  // global (cin, cout, 1, 2, 2)
    s_wt[(ci * 4 + tap) * COUT + co] = w[i];
  }
  __syncthreads();
  const int OY = isz.y * 2, OX = isz.x * 2;
  const size_t ipvol = (size_t)isz.z * isz.y * isz.x, opvol = (size_t)isz.z * OY * OX;
  const size_t total = (size_t)nb * opvol;
  const int ichunks = cin / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t ov = i % opvol;
    const int b = (int)(i / opvol);
    const int x = (int)(ov % OX), y = (int)((ov / OX) % OY), z = (int)(ov / ((size_t)OX * OY));
    const int tap = (y & 1) * 2 + (x & 1);
    const size_t iv = ((size_t)z * isz.y + (y >> 1)) * isz.x + (x >> 1);
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
    for (int ch = 0; ch < ichunks; ++ch) {
      float v[8];
      load8(in, ((size_t)b * ichunks + ch) * fmt_planes(parts), parts, ipvol, iv, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float* wp = &s_wt[((ch * 8 + e) * 4 + tap) * COUT];
#pragma unroll
        for (int co = 0; co < COUT; ++co) acc[co] = fmaf(v[e], wp[co], acc[co]);
      }
    }
#pragma unroll
    for (int oc = 0; oc < COUT / 8; ++oc) {
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = acc[oc * 8 + e] + __ldg(bias + oc * 8 + e);
      store8(out, ((size_t)b * (COUT / 8) + oc) * fmt_planes(parts), parts, opvol, ov, v);
    }
  }
}

// ---- 1x1x1 head + sigmoid -> planar fp32 --------------------------------------------------
__global__ void __launch_bounds__(kT)
head_sigmoid_cp8_kernel(const uint4* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                        float* __restrict__ out, int cin, int cout, int parts, int nb, size_t pvol) {
  extern __shared__ float s_hw[];
  for (int i = threadIdx.x; i < cout * cin; i += blockDim.x) s_hw[i] = w[i];
  for (int i = threadIdx.x; i < cout; i += blockDim.x) s_hw[cout * cin + i] = bias[i];
  __syncthreads();
  const size_t total = (size_t)nb * pvol;
  const int chunks = cin / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t vox = i % pvol, b = i / pvol;
    float acc[8];
    for (int co = 0; co < cout; ++co) acc[co] = s_hw[cout * cin + co];
    for (int ch = 0; ch < chunks; ++ch) {
      float v[8];
      load8(in, (b * chunks + ch) * fmt_planes(parts), parts, pvol, vox, v);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        for (int co = 0; co < cout; ++co) acc[co] = fmaf(v[e], s_hw[co * cin + ch * 8 + e], acc[co]);
    }
    for (int co = 0; co < cout; ++co) out[(b * cout + co) * pvol + vox] = __fdiv_rn(1.0f, 1.0f + expf(-acc[co]));
  }
}

// ---- fused head + sigmoid + crop + mask + blend --------------------------------------------
// One thread = one voxel of the (cropped) output patch, all output channels.
__global__ void __launch_bounds__(kT)
head_blend_cp8_kernel(const uint4* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias, int cin,
                      int cnet, int parts, Int3 ip, Int3 op, Int3 crop, const float* __restrict__ mask,
                      const PatchPos* __restrict__ patches, int nb, float* __restrict__ out, int channels, Int3 os,
                      float scale) {
  extern __shared__ float s_hw[];  // [channels][cin] + [channels]
  for (int i = threadIdx.x; i < channels * cin; i += blockDim.x) s_hw[i] = w[i];
  for (int i = threadIdx.x; i < channels; i += blockDim.x) s_hw[channels * cin + i] = bias[i];
  __syncthreads();
  const size_t ipvol = (size_t)ip.z * ip.y * ip.x, opvol = (size_t)op.z * op.y * op.x;
  const size_t out_vol = (size_t)os.z * os.y * os.x;
  const size_t total = (size_t)nb * opvol;
  const int chunks = cin / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t ov = i % opvol;
    const int b = (int)(i / opvol);
    const int x = (int)(ov % op.x), y = (int)((ov / op.x) % op.y), z = (int)(ov / ((size_t)op.x * op.y));
    const PatchPos pp = patches[b];
    int sy = y, sx = x;
    if (pp.flags) tta_map(pp.flags, op.y, op.x, y, x, sy, sx);  // write an augmented variant back un-transformed
    const int gz = pp.oz + z, gy = pp.oy + sy, gx = pp.ox + sx;
    if (gz < 0 || gz >= os.z || gy < 0 || gy >= os.y || gx < 0 || gx >= os.x) continue;  // clipped
    const size_t iv = ((size_t)(z + crop.z) * ip.y + (y + crop.y)) * ip.x + (x + crop.x);
    float acc[8];
    for (int co = 0; co < channels; ++co) acc[co] = s_hw[channels * cin + co];
    for (int ch = 0; ch < chunks; ++ch) {
      float v[8];
      load8(in, ((size_t)b * chunks + ch) * fmt_planes(parts), parts, ipvol, iv, v);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        for (int co = 0; co < channels; ++co) acc[co] = fmaf(v[e], s_hw[co * cin + ch * 8 + e], acc[co]);
    }
    const float m = __ldg(mask + ov) * scale;
    float* dst = out + ((size_t)gz * os.y + gy) * os.x + gx;
    for (int co = 0; co < channels; ++co) acc[co] = __fdiv_rn(1.0f, 1.0f + expf(-acc[co]));
    for (int co = 0; co < channels; ++co) {
      float sig = acc[co];
      if (pp.flags & kTtaChannelSym) sig += acc[channels - 1 - co];  // reference-literal --augment
      asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst + (size_t)co * out_vol), "f"(sig * m) : "memory");
    }
  }
}

int grid_for(size_t items) {
  size_t b = (items + kT - 1) / kT;
  if (b < 1) b = 1;
  if (b > 132 * 16) b = 132 * 16;
  return (int)b;
}

}  // namespace

void launch_planar_to_cp8(const float* in, __half* out, int channels, int parts, int nb, Int3 sz, cudaStream_t s) {
  planar_to_cp8_kernel<<<grid_for((size_t)nb * (channels / 8) * vol(sz)), kT, 0, s>>>(in, reinterpret_cast<uint4*>(out),
                                                                                     channels, parts, nb, (size_t)vol(sz));
  CFB_LAUNCH_CHECK();
}

void launch_cp8_to_planar(const __half* in, float* out, int channels, int parts, int nb, Int3 sz, cudaStream_t s) {
  cp8_to_planar_kernel<<<grid_for((size_t)nb * (channels / 8) * vol(sz)), kT, 0, s>>>(reinterpret_cast<const uint4*>(in), out,
                                                                                     channels, parts, nb, (size_t)vol(sz));
  CFB_LAUNCH_CHECK();
}

void launch_first_conv_cp8(const void* chunk, int in_dtype, Int3 cs, const PatchPos* patches, int nb, Int3 ps,
                           const float* w, const float* bias, __half* out, int parts, cudaStream_t s, const FirstConvW* cw) {
  const int tiles_x = ceil_div(ps.x, kFX), tiles_y = ceil_div(ps.y, kFY);
  dim3 grid(tiles_x * tiles_y, ps.z, nb);
  if (cw) {
    if (in_dtype == CFB_DTYPE_U8)
      first_conv_cp8_const_kernel<0><<<grid, kT, 0, s>>>(chunk, cs, patches, ps, *cw, reinterpret_cast<uint4*>(out), parts, tiles_x);
    else
      first_conv_cp8_const_kernel<1><<<grid, kT, 0, s>>>(chunk, cs, patches, ps, *cw, reinterpret_cast<uint4*>(out), parts, tiles_x);
    CFB_LAUNCH_CHECK();
    return;
  }
  if (in_dtype == CFB_DTYPE_U8)
    first_conv_cp8_kernel<0><<<grid, kT, 0, s>>>(chunk, cs, patches, ps, w, bias, reinterpret_cast<uint4*>(out), parts, tiles_x);
  else
    first_conv_cp8_kernel<1><<<grid, kT, 0, s>>>(chunk, cs, patches, ps, w, bias, reinterpret_cast<uint4*>(out), parts, tiles_x);
  CFB_LAUNCH_CHECK();
}

void launch_first_conv_cp8_from_patches(const float* patches, int nb, Int3 ps, const float* w, const float* bias,
                                        __half* out, int parts, cudaStream_t s) {
  const int tiles_x = ceil_div(ps.x, kFX), tiles_y = ceil_div(ps.y, kFY);
  dim3 grid(tiles_x * tiles_y, ps.z, nb);
  first_conv_cp8_kernel<2><<<grid, kT, 0, s>>>(patches, Int3{0, 0, 0}, nullptr, ps, w, bias, reinterpret_cast<uint4*>(out),
                                               parts, tiles_x);
  CFB_LAUNCH_CHECK();
}

void launch_maxpool_cp8(const __half* in, __half* out, int channels, int parts, int nb, Int3 isz, cudaStream_t s) {
  const size_t pc = (size_t)nb * (channels / 8);
  maxpool_cp8_kernel<<<grid_for(pc * isz.z * (isz.y / 2) * (isz.x / 2)), kT, 0, s>>>(
      reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), parts, pc, isz);
  CFB_LAUNCH_CHECK();
}

void launch_convT_cp8(const __half* in, const float* w, const float* bias, __half* out, int cin, int cout, int parts,
                      int nb, Int3 isz, cudaStream_t s) {
  const size_t items = (size_t)nb * isz.z * isz.y * 2 * isz.x * 2;
  const size_t smem = (size_t)cin * cout * 4 * sizeof(float);
  auto in16 = reinterpret_cast<const uint4*>(in);
  auto out16 = reinterpret_cast<uint4*>(out);
  if (cout == 32) {
    convT_cp8_kernel<32><<<grid_for(items), kT, smem, s>>>(in16, w, bias, out16, cin, parts, nb, isz);
  } else if (cout == 16) {
    convT_cp8_kernel<16><<<grid_for(items), kT, smem, s>>>(in16, w, bias, out16, cin, parts, nb, isz);
  } else {
    throw std::runtime_error("convT_cp8: unsupported cout");
  }
  CFB_LAUNCH_CHECK();
}

void launch_head_blend_cp8(const __half* in, const float* w, const float* bias, int cin, int cnet, int parts, Int3 ip,
                           Int3 op, Int3 crop, const float* mask, const PatchPos* patches, int nb, float* out, int channels,
                           Int3 os, float scale, cudaStream_t s) {
  if (channels > 8 || channels > cnet) throw std::runtime_error("head_blend: bad channel count");
  const size_t smem = (size_t)(channels * cin + channels) * sizeof(float);
  // only the first `channels` rows of the head are evaluated (reference patch/base.py:70-74 keeps the first N)
  head_blend_cp8_kernel<<<grid_for((size_t)nb * vol(op)), kT, smem, s>>>(reinterpret_cast<const uint4*>(in), w, bias, cin, cnet,
                                                                        parts, ip, op, crop, mask, patches, nb, out, channels, os, scale);
  CFB_LAUNCH_CHECK();
}

void launch_head_sigmoid_cp8(const __half* in, const float* w, const float* bias, float* out, int cin, int cout, int parts,
                             int nb, Int3 sz, cudaStream_t s) {
  if (cout > 8) throw std::runtime_error("head: at most 8 output channels");
  const size_t smem = (size_t)(cout * cin + cout) * sizeof(float);
  head_sigmoid_cp8_kernel<<<grid_for((size_t)nb * vol(sz)), kT, smem, s>>>(reinterpret_cast<const uint4*>(in), w, bias, out,
                                                                           cin, cout, parts, nb, (size_t)vol(sz));
  CFB_LAUNCH_CHECK();
}

}  // namespace cfb
