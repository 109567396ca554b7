// HBM-bound kernels of the inference hot path (sm_90a).  See kernels_memory.cuh.
#include "kernels_memory.cuh"

#include <algorithm>

#include "chunkflow_b200.h"

namespace cfb {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float u8_to_unit(unsigned int v) {
  // numpy: x.astype(float32); x /= 255  -> IEEE fp32 division (not a reciprocal multiply)
  return __fdiv_rn((float)v, 255.0f);
}

// max that propagates NaN (fmaxf drops it)
__device__ __forceinline__ float nan_max(float a, float b) { return (b > a || b != b) ? b : a; }

__device__ __forceinline__ void red_add_f32(float* addr, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}

__device__ __forceinline__ void red_add_v4_f32(float* addr, float4 v) {
  // one 16-byte reduction per thread: the L2 performs the read-modify-write
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// ---- extract -------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
extract_patches_kernel(const T* __restrict__ chunk, Int3 cs, const PatchPos* __restrict__ patches, int nb,
                       Int3 p, float* __restrict__ out) {
  const int qx = p.x >> 2;  // quads per row
  const int64_t total = (int64_t)nb * p.z * p.y * qx;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int xq = (int)(i % qx);
    int64_t r = i / qx;
    int y = (int)(r % p.y);
    r /= p.y;
    int z = (int)(r % p.z);
    int b = (int)(r / p.z);
    const PatchPos pp = patches[b];
    const T* src = chunk + ((int64_t)(pp.iz + z) * cs.y + (pp.iy + y)) * cs.x + pp.ix + xq * 4;
    float4 v;
    if (pp.flags) {  // test-time augmentation variant: gather through the coordinate map
      float e[4];
      for (int k = 0; k < 4; ++k) {
        int sy, sx;
        tta_map(pp.flags, p.y, p.x, y, xq * 4 + k, sy, sx);
        const T raw = chunk[((int64_t)(pp.iz + z) * cs.y + (pp.iy + sy)) * cs.x + pp.ix + sx];
        if constexpr (sizeof(T) == 1) e[k] = u8_to_unit(raw); else e[k] = raw;
      }
      v = make_float4(e[0], e[1], e[2], e[3]);
    } else if constexpr (sizeof(T) == 1) {
      if ((reinterpret_cast<uintptr_t>(src) & 3) == 0) {
        unsigned int w = __ldg(reinterpret_cast<const unsigned int*>(src));
        v = make_float4(u8_to_unit(w & 0xff), u8_to_unit((w >> 8) & 0xff), u8_to_unit((w >> 16) & 0xff),
                        u8_to_unit(w >> 24));
      } else {
        v = make_float4(u8_to_unit(__ldg(src)), u8_to_unit(__ldg(src + 1)), u8_to_unit(__ldg(src + 2)),
                        u8_to_unit(__ldg(src + 3)));
      }
    } else {
      v = make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3));
    }
    reinterpret_cast<float4*>(out)[i] = v;
  }
}

// ---- blend ---------------------------------------------------------------------------
// One thread = 4 consecutive x voxels of one output patch, all channels.
__global__ void __launch_bounds__(kThreads)
blend_patches_kernel(const float* __restrict__ net, int cnet, Int3 ip, Int3 op, Int3 crop,
                     const float* __restrict__ mask, const PatchPos* __restrict__ patches, int nb,
                     float* __restrict__ out, int channels, Int3 os, float scale) {
  const int qx = (op.x + 3) >> 2;
  const int64_t total = (int64_t)nb * op.z * op.y * qx;
  const int64_t in_vol = (int64_t)ip.z * ip.y * ip.x;
  const int64_t out_vol = (int64_t)os.z * os.y * os.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int xq = (int)(i % qx);
    int64_t r = i / qx;
    int y = (int)(r % op.y);
    r /= op.y;
    int z = (int)(r % op.z);
    int b = (int)(r / op.z);
    const PatchPos pp = patches[b];
    const int x = xq * 4;
    const int nx = min(4, op.x - x);
    if (pp.flags) {  // augmented variant: scatter back through the coordinate map, element by element
      const int gz = pp.oz + z;
      if (gz < 0 || gz >= os.z) continue;
      for (int k = 0; k < nx; ++k) {
        int sy, sx;
        tta_map(pp.flags, op.y, op.x, y, x + k, sy, sx);
        const int gy = pp.oy + sy, gx = pp.ox + sx;
        if (gy < 0 || gy >= os.y || gx < 0 || gx >= os.x) continue;
        const float mk = mask ? __ldg(mask + ((int64_t)z * op.y + y) * op.x + x + k) : 1.f;
        const float* sp = net + (int64_t)b * cnet * in_vol + ((int64_t)(z + crop.z) * ip.y + (y + crop.y)) * ip.x + (x + k + crop.x);
        float* dp = out + ((int64_t)gz * os.y + gy) * os.x + gx;
        for (int c = 0; c < channels; ++c) {
          float v = sp[(int64_t)c * in_vol];
          if (pp.flags & kTtaChannelSym) v += sp[(int64_t)(channels - 1 - c) * in_vol];  // + the channel-reversed copy
          red_add_f32(dp + (int64_t)c * out_vol, v * scale * mk);
        }
      }
      continue;
    }
    const int gz = pp.oz + z, gy = pp.oy + y, gx = pp.ox + x;
    if (gz < 0 || gz >= os.z || gy < 0 || gy >= os.y) continue;  // clipped (chunk/base.py:793-796)
    const float* m = mask ? mask + ((int64_t)z * op.y + y) * op.x + x : nullptr;
    const float* src = net + (int64_t)b * cnet * in_vol +
                       ((int64_t)(z + crop.z) * ip.y + (y + crop.y)) * ip.x + (x + crop.x);
    float* dst = out + ((int64_t)gz * os.y + gy) * os.x + gx;
    const bool vec = nx == 4 && gx >= 0 && gx + 4 <= os.x &&
                     ((reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(src) |
                       reinterpret_cast<uintptr_t>(dst) | (uintptr_t)(in_vol * 4) | (uintptr_t)(out_vol * 4)) &
                      15) == 0;
    if (vec) {
      const float4 mv = m ? __ldg(reinterpret_cast<const float4*>(m)) : make_float4(1.f, 1.f, 1.f, 1.f);
      for (int c = 0; c < channels; ++c) {
        float4 v = __ldcs(reinterpret_cast<const float4*>(src + (int64_t)c * in_vol));
        v.x = v.x * scale * mv.x;
        v.y = v.y * scale * mv.y;
        v.z = v.z * scale * mv.z;
        v.w = v.w * scale * mv.w;
        red_add_v4_f32(dst + (int64_t)c * out_vol, v);
      }
    } else {
      for (int k = 0; k < nx; ++k) {
        if (gx + k < 0 || gx + k >= os.x) continue;
        const float mk = m ? __ldg(m + k) : 1.f;
        for (int c = 0; c < channels; ++c)
          red_add_f32(dst + (int64_t)c * out_vol + k, src[(int64_t)c * in_vol + k] * scale * mk);
      }
    }
  }
}

// ---- identity backend ----------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
identity_blend_kernel(const T* __restrict__ chunk, Int3 cs, Int3 ip, Int3 op, Int3 crop,
                      const float* __restrict__ mask, const PatchPos* __restrict__ patches, int nb,
                      float* __restrict__ out, int channels, Int3 os) {
  const int64_t total = (int64_t)nb * op.z * op.y * op.x;
  const int64_t out_vol = (int64_t)os.z * os.y * os.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)(i % op.x);
    int64_t r = i / op.x;
    int y = (int)(r % op.y);
    r /= op.y;
    int z = (int)(r % op.z);
    int b = (int)(r / op.z);
    const PatchPos pp = patches[b];
    const int gz = pp.oz + z, gy = pp.oy + y, gx = pp.ox + x;
    if (gz < 0 || gz >= os.z || gy < 0 || gy >= os.y || gx < 0 || gx >= os.x) continue;
    const T raw = chunk[((int64_t)(pp.iz + z + crop.z) * cs.y + (pp.iy + y + crop.y)) * cs.x + pp.ix + x + crop.x];
    float v;
    if constexpr (sizeof(T) == 1) v = u8_to_unit(raw); else v = raw;
    v *= mask[((int64_t)z * op.y + y) * op.x + x];
    float* dst = out + ((int64_t)gz * os.y + gy) * os.x + gx;
    for (int c = 0; c < channels; ++c) red_add_f32(dst + (int64_t)c * out_vol, v);
  }
}

// ---- plugin-level crop + mask ----------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
crop_mask_kernel(const float* __restrict__ net, int cnet, Int3 ip, Int3 op, Int3 crop,
                 const float* __restrict__ mask, int nb, float* __restrict__ out, int channels, int repeat) {
  const int64_t ovol = (int64_t)op.z * op.y * op.x, ivol = (int64_t)ip.z * ip.y * ip.x;
  const int64_t total = (int64_t)nb * channels * ovol;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t v = i % ovol;
    int64_t r = i / ovol;
    int c = (int)(r % channels);
    int b = (int)(r / channels);
    int x = (int)(v % op.x);
    int y = (int)((v / op.x) % op.y);
    int z = (int)(v / ((int64_t)op.x * op.y));
    const float s = net[((int64_t)b * cnet + (repeat ? 0 : c)) * ivol +
                        ((int64_t)(z + crop.z) * ip.y + (y + crop.y)) * ip.x + (x + crop.x)];
    out[i] = s * mask[v];
  }
}

// ---- weight volume -------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
weight_volume_kernel(const float* __restrict__ mask, Int3 op, const int* __restrict__ cover_z,
                     const int* __restrict__ cover_y, const int* __restrict__ cover_x,
                     const int* __restrict__ oz0, const int* __restrict__ oy0, const int* __restrict__ ox0,
                     Int3 os, float* __restrict__ w, bool invert, int z_begin, int nz) {
  // planes [z_begin, z_begin + nz) of the volume; w holds those planes only
  const int64_t total = (int64_t)nz * os.y * os.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)(i % os.x);
    int64_t r = i / os.x;
    int y = (int)(r % os.y);
    int z = z_begin + (int)(r / os.y);
    float acc = 0.0f;  // patch-list order: z-major, then y, then x -> same fp32 sum as numpy's +=
    for (int a = 0; a < kMaxCover; ++a) {
      int pz = cover_z[z * kMaxCover + a];
      if (pz < 0) break;
      int lz = z - oz0[pz];
      for (int bb = 0; bb < kMaxCover; ++bb) {
        int py = cover_y[y * kMaxCover + bb];
        if (py < 0) break;
        int ly = y - oy0[py];
        for (int c = 0; c < kMaxCover; ++c) {
          int px = cover_x[x * kMaxCover + c];
          if (px < 0) break;
          int lx = x - ox0[px];
          acc += __ldg(mask + ((int64_t)lz * op.y + ly) * op.x + lx);
        }
      }
    }
    w[i] = invert ? __fdiv_rn(1.0f, acc) : acc;
  }
}

// ---- normalise -----------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
normalize_kernel(float* __restrict__ out, const float* __restrict__ w, bool w_is_inverse, int channels,
                 int64_t nvox, int64_t cstride, unsigned int* __restrict__ max_bits,
                 const unsigned int* __restrict__ nonzero_flag) {
  const bool force_zero = nonzero_flag != nullptr && *nonzero_flag == 0u;
  float vmax = 0.0f;
  const int64_t nq = nvox >> 2;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w)) & 15) == 0 && (nvox & 3) == 0 &&
                      (cstride & 3) == 0;
  if (vec_ok) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nq;
         i += (int64_t)gridDim.x * blockDim.x) {
      float4 s = make_float4(1.f, 1.f, 1.f, 1.f);
      if (w != nullptr) {
        s = __ldcs(reinterpret_cast<const float4*>(w) + i);
        if (!w_is_inverse) s = make_float4(__fdiv_rn(1.f, s.x), __fdiv_rn(1.f, s.y), __fdiv_rn(1.f, s.z), __fdiv_rn(1.f, s.w));
      }
      for (int c = 0; c < channels; ++c) {
        float4* p = reinterpret_cast<float4*>(out + (int64_t)c * cstride) + i;
        float4 v = *p;
        v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
        if (force_zero) v = make_float4(0.f, 0.f, 0.f, 0.f);
        vmax = nan_max(nan_max(vmax, nan_max(v.x, v.y)), nan_max(v.z, v.w));
        __stcs(p, v);
      }
    }
  } else {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvox;
         i += (int64_t)gridDim.x * blockDim.x) {
      float s = 1.f;
      if (w != nullptr) s = w_is_inverse ? w[i] : __fdiv_rn(1.f, w[i]);
      for (int c = 0; c < channels; ++c) {
        float v = out[(int64_t)c * cstride + i] * s;
        if (force_zero) v = 0.f;
        vmax = nan_max(vmax, v);
        out[(int64_t)c * cstride + i] = v;
      }
    }
  }
  // NaN must not slip through the range check (the reference's assert_array_less raises on NaN): nan_max keeps it,
  // and a quiet-NaN bit pattern (0x7fc00000) is larger than the bits of every finite positive float
  for (int o = 16; o > 0; o >>= 1) vmax = nan_max(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
  if ((threadIdx.x & 31) == 0 && max_bits != nullptr && !(vmax <= 0.f))
    atomicMax(max_bits, vmax != vmax ? 0x7fc00000u : __float_as_uint(vmax));
}

__global__ void __launch_bounds__(kThreads)
myelin_mask_kernel(float* __restrict__ out, int channels, int64_t nvox, float thr) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvox;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float keep = out[(int64_t)(channels - 1) * nvox + i] < thr ? 1.f : 0.f;
    for (int c = 0; c < channels - 1; ++c) out[(int64_t)c * nvox + i] *= keep;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
any_nonzero_kernel(const T* __restrict__ p, int64_t n, unsigned int* __restrict__ flag) {
  bool nz = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    nz |= (p[i] != T(0));
  if (__any_sync(0xffffffffu, nz) && (threadIdx.x & 31) == 0) atomicOr(flag, 1u);
}

int grid_for(int64_t items, int max_blocks = 132 * 16) {
  int64_t b = ceil_div64(items, kThreads);
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

}  // namespace

void launch_extract_patches(const void* chunk, int in_dtype, Int3 cs, const PatchPos* patches, int nb,
                            Int3 p, float* out, cudaStream_t s) {
  const int64_t items = (int64_t)nb * p.z * p.y * (p.x / 4);
  if (in_dtype == CFB_DTYPE_U8)
    extract_patches_kernel<uint8_t><<<grid_for(items), kThreads, 0, s>>>((const uint8_t*)chunk, cs, patches, nb, p, out);
  else
    extract_patches_kernel<float><<<grid_for(items), kThreads, 0, s>>>((const float*)chunk, cs, patches, nb, p, out);
  CFB_LAUNCH_CHECK();
}

void launch_blend_patches(const float* net, int cnet, Int3 ip, Int3 op, Int3 crop, const float* mask,
                          const PatchPos* patches, int nb, float* out, int channels, Int3 os, float scale,
                          cudaStream_t s) {
  const int64_t items = (int64_t)nb * op.z * op.y * ((op.x + 3) / 4);
  blend_patches_kernel<<<grid_for(items), kThreads, 0, s>>>(net, cnet, ip, op, crop, mask, patches, nb, out,
                                                            channels, os, scale);
  CFB_LAUNCH_CHECK();
}

void launch_identity_blend(const void* chunk, int in_dtype, Int3 cs, Int3 ip, Int3 op, Int3 crop,
                           const float* mask, const PatchPos* patches, int nb, float* out, int channels,
                           Int3 os, cudaStream_t s) {
  const int64_t items = (int64_t)nb * op.z * op.y * op.x;
  if (in_dtype == CFB_DTYPE_U8)
    identity_blend_kernel<uint8_t><<<grid_for(items), kThreads, 0, s>>>((const uint8_t*)chunk, cs, ip, op, crop,
                                                                        mask, patches, nb, out, channels, os);
  else
    identity_blend_kernel<float><<<grid_for(items), kThreads, 0, s>>>((const float*)chunk, cs, ip, op, crop, mask,
                                                                      patches, nb, out, channels, os);
  CFB_LAUNCH_CHECK();
}

void launch_crop_mask(const float* net, int cnet, Int3 ip, Int3 op, Int3 crop, const float* mask, int nb, float* out,
                      int channels, bool repeat, cudaStream_t s) {
  crop_mask_kernel<<<grid_for((int64_t)nb * channels * vol(op)), kThreads, 0, s>>>(net, cnet, ip, op, crop, mask, nb, out,
                                                                                   channels, repeat ? 1 : 0);
  CFB_LAUNCH_CHECK();
}

void launch_weight_volume(const float* mask, Int3 op, const int* cover_z, const int* cover_y, const int* cover_x,
                          const int* oz0, const int* oy0, const int* ox0, Int3 os, float* w, bool invert,
                          cudaStream_t s, int z_begin, int z_end) {
  if (z_end < 0) z_end = os.z;
  const int nz = z_end - z_begin;
  if (nz <= 0) return;
  weight_volume_kernel<<<grid_for((int64_t)nz * os.y * os.x), kThreads, 0, s>>>(mask, op, cover_z, cover_y, cover_x, oz0, oy0, ox0,
                                                                               os, w, invert, z_begin, nz);
  CFB_LAUNCH_CHECK();
}

// dst += src (halo planes received from another rank, BASELINE config #5)
__global__ void __launch_bounds__(256) halo_add_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n) {
  const int64_t nq = n >> 2;
  const bool vec = ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) == 0;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, step = (int64_t)gridDim.x * blockDim.x;
  if (vec) {
    for (int64_t i = tid; i < nq; i += step) {
      float4 a = reinterpret_cast<float4*>(dst)[i];
      const float4 b = __ldcs(reinterpret_cast<const float4*>(src) + i);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      reinterpret_cast<float4*>(dst)[i] = a;
    }
    for (int64_t i = (nq << 2) + tid; i < n; i += step) dst[i] += src[i];
  } else {
    for (int64_t i = tid; i < n; i += step) dst[i] += src[i];
  }
}

void launch_halo_add(float* dst, const float* src, int64_t n, cudaStream_t s) {
  if (n <= 0) return;
  int64_t blocks = std::min<int64_t>(ceil_div64(n / 4 + 1, 256), 132 * 16);
  halo_add_kernel<<<(int)blocks, 256, 0, s>>>(dst, src, n);
  CFB_LAUNCH_CHECK();
}

void launch_normalize(float* out, const float* w, bool w_is_inverse, int channels, int64_t nvox,
                      unsigned int* max_bits, const unsigned int* nonzero_flag, cudaStream_t s, int64_t channel_stride) {
  if (channel_stride <= 0) channel_stride = nvox;
  normalize_kernel<<<grid_for(nvox / 4 + 1), kThreads, 0, s>>>(out, w, w_is_inverse, channels, nvox, channel_stride,
                                                               max_bits, nonzero_flag);
  CFB_LAUNCH_CHECK();
}

void launch_myelin_mask(float* out, int channels, int64_t nvox, float threshold, cudaStream_t s) {
  myelin_mask_kernel<<<grid_for(nvox), kThreads, 0, s>>>(out, channels, nvox, threshold);
  CFB_LAUNCH_CHECK();
}

void launch_any_nonzero(const void* chunk, int in_dtype, int64_t n, unsigned int* flag, cudaStream_t s) {
  if (in_dtype == CFB_DTYPE_U8) {
    // scan 16 bytes per thread where alignment allows
    if ((reinterpret_cast<uintptr_t>(chunk) & 15) == 0 && (n & 15) == 0)
      any_nonzero_kernel<unsigned long long><<<grid_for(n / 8), kThreads, 0, s>>>((const unsigned long long*)chunk, n / 8, flag);
    else
      any_nonzero_kernel<uint8_t><<<grid_for(n), kThreads, 0, s>>>((const uint8_t*)chunk, n, flag);
  } else {
    any_nonzero_kernel<float><<<grid_for(n), kThreads, 0, s>>>((const float*)chunk, n, flag);
  }
  CFB_LAUNCH_CHECK();
}

}  // namespace cfb
