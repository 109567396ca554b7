// "f16f8" activation / weight number format of the wgmma convolution stack (precision mode CFB_PRECISION_F16F8_UMMA).
//
// The f16x3 mode spends THREE tensor-core products per multiply (a_hi w_hi + a_hi w_lo + a_lo w_hi, all fp16).  The two
// correction terms are 2^-11 of the main one, so they need only a few significant bits themselves: here they run as ONE
// fp8 (e4m3) product of twice the K depth -- kind::f8f6f4, K = 32 = [a | a_lo] x [w_lo ; w] -- at the price of one fp16
// MMA, i.e. TWO tensor-core products per multiply instead of three, accumulating in the same fp32 accumulators:
//
//     acc  =  H * WH            (kind::f16,    K = 16 channels)
//          +  A8 * WL8 + L8 * W8 (kind::f8f6f4, K = 32 = 16 channels x {A8, L8})
//
//     H   = fp16(a * alpha)            L   = a * alpha - H          (exact in fp32, |L| <= 2^-11 |a alpha|)
//     A8  = e4m3(a * gamma)            L8  = e4m3(L * lambda)
//     WH  = fp16(w * beta)             WL  = w * beta - WH
//     W8  = e4m3(w * delta)            WL8 = e4m3(WL * mu)
//
// with powers of two chosen such that every term carries the scale alpha * beta:  gamma * mu = alpha and
// lambda * delta = beta.  e4m3 spans 2^-9 .. 448, fp16 6e-8 .. 65504:
//     alpha = 32, gamma = 1, lambda = 64, mu = 32         (activations: full accuracy up to |a| = 448, graceful --
//                                                           fp16-level corrections -- up to 2047, clamped beyond)
//     beta  = 2^14 / wmax', delta = beta / 64              (per layer, wmax' = max |w| rounded up to a power of two)
// The epilogue multiplies the accumulator by 1 / (alpha * beta).  Error of one product: the dropped a_lo w_lo (2^-24) plus
// the e4m3 rounding (2^-4 relative) of two terms that are 2^-12 of the product: ~2^-16 worst case, ~2^-17.5 rms; the
// tests assert the whole network within 5e-4 max-abs of the fp32 reference.
//
// HBM layout ("CP8", kernels_conv.cuh) is unchanged: planes of 16-byte voxel records, plane = chunk * 2 + part for
// 8-channel chunk `chunk`.  Per K step (two chunks c0 = 2k, c1 = 2k + 1, i.e. channels 16k .. 16k + 15):
//     (c0, part 0) = H  channels 0..7      (c1, part 0) = H  channels 8..15      (fp16 x 8)
//     (c0, part 1) = A8 channels 0..15     (c1, part 1) = L8 channels 0..15      (e4m3 x 16)
// so the fp16 A tile of a K step is planes (c0,0),(c1,0) and the fp8 A tile (K = 32) is planes (c0,1),(c1,1): exactly the
// addresses of the hi and lo tiles of the f16x3 mode.
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <cstdint>

namespace cfb {

constexpr float kActAlpha = 32.0f;    // H  = fp16(a * alpha)
constexpr float kActGamma = 1.0f;     // A8 = e4m3(a * gamma)
constexpr float kActLambda = 64.0f;   // L8 = e4m3(L * lambda)
constexpr float kWgtMu = 32.0f;       // WL8 = e4m3(WL * mu),  gamma * mu = alpha
constexpr float kHalfMax = 65504.0f;

// activation number formats of the CP8 tensors
enum ActFmt : int { kFmtF16 = 1, kFmtF16x2 = 2, kFmtF16F8 = 3 };
__host__ __device__ constexpr int fmt_planes(int fmt) { return fmt == kFmtF16 ? 1 : 2; }  // planes per 8-channel chunk

__device__ __forceinline__ uint32_t af_pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t af_pack_e4m3x4(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
__device__ __forceinline__ void af_unpack_e4m3x4(uint32_t u, float (&v)[4]) {
  const __half2_raw a = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(u & 0xffffu), __NV_E4M3);
  const __half2_raw b = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(u >> 16), __NV_E4M3);
  const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&a)), fb = __half22float2(*reinterpret_cast<const __half2*>(&b));
  v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}

// 16 channels of one voxel (one K step) -> the four 16-byte records (H 0..7, H 8..15, A8 0..15, L8 0..15).
// Per channel pair: one packed f16x2 conversion, its two widenings, and the residual as ONE fma each
// (L * lambda = a * (alpha lambda) - H * lambda, exact: the products are power-of-two scalings).
__device__ __forceinline__ void af_encode16(const float (&v)[16], uint4& h0, uint4& h1, uint4& a8, uint4& l8) {
  uint32_t hw[8];
  float l[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float s0 = fminf(fmaxf(v[2 * i] * kActAlpha, -kHalfMax), kHalfMax), s1 = fminf(fmaxf(v[2 * i + 1] * kActAlpha, -kHalfMax), kHalfMax);
    const __half2 h = __floats2half2_rn(s0, s1);
    const float2 f = __half22float2(h);
    hw[i] = *reinterpret_cast<const uint32_t*>(&h);
    l[2 * i] = fmaf(f.x, -kActLambda, s0 * kActLambda);
    l[2 * i + 1] = fmaf(f.y, -kActLambda, s1 * kActLambda);
  }
  h0 = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  h1 = make_uint4(hw[4], hw[5], hw[6], hw[7]);
  a8 = make_uint4(af_pack_e4m3x4(v[0] * kActGamma, v[1] * kActGamma, v[2] * kActGamma, v[3] * kActGamma),
                  af_pack_e4m3x4(v[4] * kActGamma, v[5] * kActGamma, v[6] * kActGamma, v[7] * kActGamma),
                  af_pack_e4m3x4(v[8] * kActGamma, v[9] * kActGamma, v[10] * kActGamma, v[11] * kActGamma),
                  af_pack_e4m3x4(v[12] * kActGamma, v[13] * kActGamma, v[14] * kActGamma, v[15] * kActGamma));
  l8 = make_uint4(af_pack_e4m3x4(l[0], l[1], l[2], l[3]), af_pack_e4m3x4(l[4], l[5], l[6], l[7]),
                  af_pack_e4m3x4(l[8], l[9], l[10], l[11]), af_pack_e4m3x4(l[12], l[13], l[14], l[15]));
}

// value of 8 channels from their H record and the matching half (2 words) of the L8 record
__device__ __forceinline__ void af_decode8(const uint4& h, uint32_t l8a, uint32_t l8b, float (&v)[8]) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&h.y)),
               c = __half22float2(*reinterpret_cast<const __half2*>(&h.z)), d = __half22float2(*reinterpret_cast<const __half2*>(&h.w));
  float la[4], lb[4];
  af_unpack_e4m3x4(l8a, la);
  af_unpack_e4m3x4(l8b, lb);
  constexpr float il = 1.0f / kActLambda, ia = 1.0f / kActAlpha;
  v[0] = (a.x + la[0] * il) * ia; v[1] = (a.y + la[1] * il) * ia; v[2] = (b.x + la[2] * il) * ia; v[3] = (b.y + la[3] * il) * ia;
  v[4] = (c.x + lb[0] * il) * ia; v[5] = (c.y + lb[1] * il) * ia; v[6] = (d.x + lb[2] * il) * ia; v[7] = (d.y + lb[3] * il) * ia;
}

}  // namespace cfb
