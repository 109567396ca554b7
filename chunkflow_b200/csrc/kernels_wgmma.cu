// wgmma / TMA implicit-GEMM 3x3x3 convolution for sm_90a.  See kernels_conv.cuh for the activation
// layout.  One CTA owns a (batch, y-tile, x-tile) column of the patch and marches along z with a ring
// of three z-planes in shared memory:
//
//   warp 0       : A producer  -- one TMA box per z-plane (halo rows/cols, zero fill outside the patch)
//   warp 1       : B producer  -- the packed weights of one tap per stage via cp.async.bulk
//   warpgroups 1, 2: consumers -- per z-plane job: 27 taps x K steps x (up to MT) tiles of wgmma.mma_async
//                                 (M = 64 positions, N = Cout or 2 * Cout, fp32 accumulators in registers),
//                                 then the epilogue: bias, ReLU, number format, 16-byte stores
//
// A tile is a dense run of 64 positions of the (TY + 2) x pitch halo plane; a tap (dy, dx) is a plain
// +16 B x (dy * pitch + dx) on the descriptor start address.  Positions in the two halo columns of a row
// compute junk that the epilogue drops.
//
// Number formats (act_format.cuh), all accumulating in fp32:
//   f16   : acc = A * W                                  (one fp16 product)
//   f16x2 : acc = A_hi * [W_hi | W_lo] + A_lo * W_hi     (N = 2 Cout for the first product; the halves are added)
//   f16f8 : acc = H * WH + [A8 | L8] * [WL8 ; W8]        (fp16 K = 16 plus e4m3 K = 32 into a second accumulator half),
//           scaled by 1 / (alpha beta)
#include "kernels_wgmma.cuh"

namespace cfb {

namespace {

template <int FMT>
void dispatch(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb, Int3 sz,
              bool relu, cudaStream_t s, const ConvTail* tail, __half* pool_out) {
  const int cin = ca + cb, cout = w.cout;
#define CFB_CASE(CI, CO) \
  if (cin == CI && cout == CO) return launch_cfg<CI, CO, FMT, kConv>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail);
  if (pool_out) {  // the two encoder layers that feed a pool
    if (cin == 16 && cout == 16) return launch_cfg<16, 16, FMT, kConvPool>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr, pool_out);
    if (cin == 32 && cout == 32) return launch_cfg<32, 32, FMT, kConvPool>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr, pool_out);
    if (launch_conv3_wgmma_wide(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, pool_out)) return;
    throw std::runtime_error("conv3_wgmma: fused pooling exists for the 16->16, 32->32 and 64->64 layers");
  }
  CFB_CASE(16, 16) CFB_CASE(16, 32) CFB_CASE(32, 32) CFB_CASE(32, 64) CFB_CASE(64, 64) CFB_CASE(64, 32) CFB_CASE(32, 16)
#undef CFB_CASE
  if (!tail && launch_conv3_wgmma_wide(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr)) return;
  throw std::runtime_error("conv3_wgmma: unsupported channel configuration " + std::to_string(cin) + "->" + std::to_string(cout));
}

}  // namespace

void launch_conv3_wgmma(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb,
                        Int3 sz, bool relu, cudaStream_t s, const ConvTail* tail, __half* pool_out) {
  if (ca % 16 || (cb % 16) || w.cin != ca + cb || w.taps != 27) throw std::runtime_error("conv3_wgmma: channel mismatch");
  if (pool_out && (tail || (sz.y & 1) || (sz.x & 1))) throw std::runtime_error("conv3_wgmma: pooling needs even y, x and no fused tail");
  if (tail && tail->channels > 8) throw std::runtime_error("fused tail: at most 8 channels");
  if (w.fmt == kFmtF16F8) dispatch<kFmtF16F8>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail, pool_out);
  else if (w.fmt == kFmtF16x2) dispatch<kFmtF16x2>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail, pool_out);
  else dispatch<kFmtF16>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail, pool_out);
}

void launch_convT_wgmma(const __half* in, const PackedConv& w, __half* out, int nb, Int3 in_size, cudaStream_t s) {
  if (w.taps != 4) throw std::runtime_error("convT_wgmma: weights are not a (1,2,2) transposed convolution");
#define CFB_CASE(CI, CO)                                                                                                   \
  if (w.cin == CI && w.cout == CO) {                                                                                       \
    if (w.fmt == kFmtF16F8) return launch_cfg<CI, CO, kFmtF16F8, kConvT>(in, CI, nullptr, 0, w, out, nb, in_size, false, s, nullptr); \
    if (w.fmt == kFmtF16x2) return launch_cfg<CI, CO, kFmtF16x2, kConvT>(in, CI, nullptr, 0, w, out, nb, in_size, false, s, nullptr); \
    return launch_cfg<CI, CO, kFmtF16, kConvT>(in, CI, nullptr, 0, w, out, nb, in_size, false, s, nullptr);                \
  }
  CFB_CASE(64, 32) CFB_CASE(32, 16)
#undef CFB_CASE
  if (launch_convT_wgmma_wide(in, w, out, nb, in_size, s)) return;
  throw std::runtime_error("convT_wgmma: unsupported channel configuration");
}

// ------------------------------------------------------------------------------------------
// Weight packing (host)
// ------------------------------------------------------------------------------------------
// power of two >= the largest |w| of a layer (f16f8 mode: beta = 2^14 / wmax', act_format.cuh)
static float weight_beta(const float* w, size_t n) {
  float wmax = 0.f;
  for (size_t i = 0; i < n; ++i) wmax = std::max(wmax, std::fabs(w[i]));
  if (!(wmax > 0.f) || !std::isfinite(wmax)) return 16384.0f;
  return 16384.0f / std::exp2(std::ceil(std::log2(wmax)));
}
static uint8_t to_e4m3(float v) { return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3); }

// One block per (tap, K step of 16 input channels), BLK = parts * 32 * cout bytes, rows are output channels,
// [chunk of 8 input channels][rows][16 bytes] (K-major core matrices):
//   f16   : [2][cout]      fp16(w)
//   f16x2 : [2][2 cout]    rows 0..cout-1 fp16(w), rows cout..2cout-1 fp16(w - fp16(w))
//   f16f8 : [2][cout] fp16(w beta), then [2][cout] x 16 e4m3: chunk 0 = WL8 = e4m3((w beta - WH) mu),
//           chunk 1 = W8 = e4m3(w delta) of the same 16 input channels
// `W(co, ci, tap)` reads the layer's fp32 weights; a transposed convolution has 4 taps (its output parities).
template <typename WF>
static void pack_blocks(WF W, const float* h_w, const float* h_bias, int cin, int cout, int taps, int fmt, PackedConv& out) {
  free_packed(out);
  const int parts = fmt_planes(fmt);
  const int KS = cin / 16;
  const size_t blk = (size_t)parts * 32 * cout;
  std::vector<uint8_t> buf((size_t)taps * KS * blk, 0);
  const float beta = fmt == kFmtF16F8 ? weight_beta(h_w, (size_t)cout * cin * taps) : 1.0f, delta = beta / kActLambda;
  auto put_half = [&](size_t off, float v) { const __half h = __float2half_rn(v); std::memcpy(&buf[off], &h, 2); };
  for (int t = 0; t < taps; ++t)
    for (int ks = 0; ks < KS; ++ks) {
      const size_t base = ((size_t)t * KS + ks) * blk;
      for (int kc = 0; kc < 2; ++kc)
        for (int co = 0; co < cout; ++co) {
          for (int e = 0; e < 8; ++e) {
            const int ci = ks * 16 + kc * 8 + e;
            const float wv = W(co, ci, t);
            if (fmt == kFmtF16) {
              put_half(base + ((size_t)kc * cout + co) * 16 + 2 * e, wv);
            } else if (fmt == kFmtF16x2) {
              const float hi = __half2float(__float2half_rn(wv));
              put_half(base + ((size_t)kc * 2 * cout + co) * 16 + 2 * e, wv);
              put_half(base + ((size_t)kc * 2 * cout + cout + co) * 16 + 2 * e, wv - hi);
            } else {
              put_half(base + ((size_t)kc * cout + co) * 16 + 2 * e, wv * beta);
            }
          }
          if (fmt == kFmtF16F8) {
            uint8_t* dst = &buf[base + (size_t)32 * cout + ((size_t)kc * cout + co) * 16];
            for (int j = 0; j < 16; ++j) {
              const float w0 = W(co, ks * 16 + j, t), wb = w0 * beta;
              dst[j] = kc ? to_e4m3(w0 * delta) : to_e4m3((wb - __half2float(__float2half_rn(wb))) * kWgtMu);
            }
          }
        }
    }
  out.cin = cin; out.cout = cout; out.parts = parts; out.fmt = fmt; out.taps = taps;
  out.acc_scale = fmt == kFmtF16F8 ? 1.0f / (kActAlpha * beta) : 1.0f;
  out.tuned = std::make_shared<std::map<uint64_t, ConvTile>>();
  out.bytes = buf.size();
  CFB_CUDA(cudaMalloc(&out.w, out.bytes));
  CFB_CUDA(cudaMemcpy(out.w, buf.data(), out.bytes, cudaMemcpyHostToDevice));
  CFB_CUDA(cudaMalloc(&out.bias, cout * sizeof(float)));
  CFB_CUDA(cudaMemcpy(out.bias, h_bias, cout * sizeof(float), cudaMemcpyHostToDevice));
}

void pack_conv3_weights(const float* h_w, const float* h_bias, int cin, int cout, int fmt, PackedConv& out) {
  if (cout > 64) {  // split along N (kernels_wgmma_wide.cu): rows [64 h, 64 h + 64) of the weights are half h
    if (cout != 128) throw std::runtime_error("conv3_wgmma: cout above 64 must be 128");
    free_packed(out);
    auto halves = std::make_shared<std::array<PackedConv, 2>>();
    for (int h = 0; h < 2; ++h) pack_conv3_weights(h_w + (size_t)h * 64 * cin * 27, h_bias + h * 64, cin, 64, fmt, (*halves)[h]);
    out.cin = cin; out.cout = cout; out.parts = fmt_planes(fmt); out.fmt = fmt; out.taps = 27;
    out.halves = halves;
    return;
  }
  pack_blocks([&](int co, int ci, int t) { return h_w[((size_t)co * cin + ci) * 27 + t]; }, h_w, h_bias, cin, cout, 27, fmt, out);
}

// h_w: (cin, cout, 1, 2, 2); tap = (oy & 1) * 2 + (ox & 1)
void pack_convT_weights(const float* h_w, const float* h_bias, int cin, int cout, int fmt, PackedConv& out) {
  pack_blocks([&](int co, int ci, int t) { return h_w[((size_t)ci * cout + co) * 4 + t]; }, h_w, h_bias, cin, cout, 4, fmt, out);
}

void free_packed(PackedConv& p) {
  if (p.halves)
    for (PackedConv& h : *p.halves) free_packed(h);
  if (p.w) cudaFree(p.w);
  if (p.bias) cudaFree(p.bias);
  p = PackedConv{};
}

}  // namespace cfb
