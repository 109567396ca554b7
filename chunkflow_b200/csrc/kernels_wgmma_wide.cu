// The wgmma convolutions that only the 4-level U-Net has (widths 16, 32, 64, 128): the 64 -> 64 layer with the fused
// (1,2,2) max pool, 128 (also the 64 + 64 decoder concat) -> 64, the transposed 128 -> 64, and 64 -> 128 and 128 -> 128
// as two halves on the 64 -> 64 and 128 -> 64 kernels.  The kernel
// template is the one of kernels_wgmma.cu (kernels_wgmma.cuh); these instantiations live in a translation unit of their own
// so that the layers of the 2- and 3-level networks keep their code exactly.
//
// The layers with 128 output channels are split along N into two 64-channel halves (pack_conv3_weights packs them as two
// layers), run as 64 -> 64 and 128 -> 64 kernels over the whole batch, each half writing its own half of the output: a
// 128-channel CP8 tensor is stored half-major (kernels_conv.cuh), and the layers that read one take its halves as the two
// sources of a concat.  One 128-wide accumulator would be 128 fp32 registers per consumer thread in the split formats
// (N = 2 Cout = 256), and ptxas spills it within the 168 registers that 384 threads leave.
#include "kernels_wgmma.cuh"

namespace cfb {

namespace {

template <int FMT>
bool conv3_wide(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb, Int3 sz,
                bool relu, cudaStream_t s, __half* pool_out) {
  const int cin = ca + cb, cout = w.cout;
  if (pool_out) {
    if (cin == 64 && cout == 64) { launch_cfg<64, 64, FMT, kConvPool>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr, pool_out); return true; }
    return false;
  }
#define CFB_CASE(CI, CO) \
  if (cin == CI && cout == CO) { launch_cfg<CI, CO, FMT, kConv>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr); return true; }
  CFB_CASE(128, 64)
#undef CFB_CASE
  return false;
}

}  // namespace

bool launch_conv3_wgmma_wide(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb,
                             Int3 sz, bool relu, cudaStream_t s, __half* pool_out) {
  const size_t half = (size_t)nb * 8 * w.parts * vol(sz) * 8;  // fp16 values of one 64-channel half of a 128-channel tensor
  if (ca == 128 && cb == 0) {  // a 128-channel tensor is stored as its two halves (kernels_conv.cuh): the concat of two sources
    srcB = srcA + half;
    ca = cb = 64;
  }
  if (w.halves && !pool_out) {
    for (int h = 0; h < 2; ++h) launch_conv3_wgmma(srcA, ca, srcB, cb, (*w.halves)[h], out + h * half, nb, sz, relu, s);
    return true;
  }
  if (w.fmt == kFmtF16F8) return conv3_wide<kFmtF16F8>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, pool_out);
  if (w.fmt == kFmtF16x2) return conv3_wide<kFmtF16x2>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, pool_out);
  return conv3_wide<kFmtF16>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, pool_out);
}

bool launch_convT_wgmma_wide(const __half* in, const PackedConv& w, __half* out, int nb, Int3 in_size, cudaStream_t s) {
  if (w.cin != 128 || w.cout != 64) return false;
  const __half* in_hi = in + (size_t)nb * 8 * w.parts * vol(in_size) * 8;  // the second half of the 128 input channels
  if (w.fmt == kFmtF16F8) launch_cfg<128, 64, kFmtF16F8, kConvT>(in, 64, in_hi, 64, w, out, nb, in_size, false, s, nullptr);
  else if (w.fmt == kFmtF16x2) launch_cfg<128, 64, kFmtF16x2, kConvT>(in, 64, in_hi, 64, w, out, nb, in_size, false, s, nullptr);
  else launch_cfg<128, 64, kFmtF16, kConvT>(in, 64, in_hi, 64, w, out, nb, in_size, false, s, nullptr);
  return true;
}

}  // namespace cfb
