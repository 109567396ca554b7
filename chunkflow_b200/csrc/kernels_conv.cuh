// wgmma / TMA implicit-GEMM 3x3x3 convolution and the fp16 "chunk-planar" activation
// layout it works on.  Declarations.
//
// Activation layout in HBM ("CP8"): (batch, C/8, P, Z, Y, X, 8) fp16 -- a tensor of 128 channels is stored half-major,
// (2, batch, 8, P, Z, Y, X, 8), each 64-channel half a CP8 tensor of its own -- where P = 1 (single
// fp16) or 2 (hi/lo split: value = hi + lo, |lo| <= ulp(hi)/2, ~22 significant bits).  One
// (chunk, part) plane is a dense (Z, Y, X, 8) array of 16-byte voxel records, so that
//   * TMA can stage a halo box of any (z, y, x) offset into shared memory with zero fill
//     outside the patch (SAME padding at the PATCH border for free), and
//   * the staged box IS the canonical no-swizzle K-major wgmma operand layout: 8 consecutive
//     voxels x 16 bytes form one core matrix, a tap shift of the 3x3x3 stencil is a plain
//     +16 B x (dy*pitch + dx) on the descriptor start address, and the second 8-channel chunk
//     of a K=16 step sits one plane further (leading byte offset).
#pragma once
#include <cuda_fp16.h>

#include <array>
#include <map>
#include <memory>

#include "act_format.cuh"
#include "common.cuh"

namespace cfb {

// One tiling of the wgmma convolution (see kernels_wgmma.cu): x tile, rows per tile, weight stages,
// output planes per CTA.
struct ConvTile {
  int XT = 0, TY = 0, pitch = 0, bstages = 0, zblk = 0;
  bool resident = false;
  double cost = 0.0;
};

// Weights of one 3x3x3 or (1,2,2)-transposed layer packed for the B operand (layout in pack_blocks, kernels_wgmma.cu).
struct PackedConv {
  void* w = nullptr;       // device, (tap, K step) blocks
  float* bias = nullptr;
  int cin = 0, cout = 0, parts = 1, taps = 0;
  int fmt = 0;             // ActFmt of the activations this layer reads and writes (act_format.cuh)
  float acc_scale = 1.0f;  // f16f8: 1 / (alpha * beta), applied to the accumulator by the epilogue
  size_t bytes = 0;
  std::shared_ptr<std::map<uint64_t, ConvTile>> tuned;  // chosen tiling per (size, batch)
  // cout 128: no blocks of its own, but the two halves of 64 output channels, each packed as a layer (kernels_wgmma_wide.cu)
  std::shared_ptr<std::array<PackedConv, 2>> halves;
};

void pack_conv3_weights(const float* h_w, const float* h_bias, int cin, int cout, int fmt, PackedConv& out);  // fmt: ActFmt
void pack_convT_weights(const float* h_w, const float* h_bias, int cin, int cout, int fmt, PackedConv& out);  // h_w: (cin, cout, 1, 2, 2)
void free_packed(PackedConv& p);

// One 3x3x3 convolution + bias + ReLU on wgmma.  Input = channel concat of srcA (ca channels)
// and srcB (cb channels, may be null); all tensors CP8 in the layer's format.
// If `tail` is given (16 -> 16 layers only) the epilogue does not store the activation but applies the
// fused network tail: 1x1x1 head + sigmoid + crop + bump mask + red.global.add into the output chunk.
// The blend steps of the other routes (network.cu) take their parameters from the same struct.
struct ConvTail {
  const float* head_w;      // device, (>= channels, 16): the first `channels` rows are evaluated
  const float* head_b;      // device
  const PatchPos* patches;  // device, this batch
  const float* mask;        // device, output patch mask (out_patch)
  float* out;               // device, (channels, out_size)
  int channels;
  Int3 out_patch, crop, out_size;
  float scale;              // 1, or 1/8 when the batch holds the 8 test-time-augmentation variants
};
// `pool_out` (16->16, 32->32 and 64->64 layers): the (1,2,2) max-pooled output, CP8 of (Z, Y/2, X/2), written by the same epilogue.
void launch_conv3_wgmma(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out,
                        int nb, Int3 size, bool relu, cudaStream_t s, const ConvTail* tail = nullptr, __half* pool_out = nullptr);
// ConvTranspose kernel = stride = (1,2,2) on wgmma: in CP8 (nb, cin) of in_size, out CP8 (nb, cout) of (Z, 2Y, 2X); no ReLU.
void launch_convT_wgmma(const __half* in, const PackedConv& w, __half* out, int nb, Int3 in_size, cudaStream_t s);

// Layout conversion (tests / debug): planar fp32 (nb, C, Z,Y,X) <-> CP8.
void launch_planar_to_cp8(const float* in, __half* out, int channels, int parts, int nb, Int3 size, cudaStream_t s);
void launch_cp8_to_planar(const __half* in, float* out, int channels, int parts, int nb, Int3 size, cudaStream_t s);

// Weights of the first layer as a kernel PARAMETER (1.8 KB in the constant bank): every FFMA takes its weight as a
// constant-bank operand, so the kernel issues no shared-memory load for weights.
struct FirstConvW {
  float w[27][16];  // [tap][cout]
  float b[16];
};

// First layer: extract `nb` patches from the uint8/f32 chunk (normalised by 1/255), 3x3x3
// convolution 1 -> 16 in fp32 on CUDA cores, ReLU, CP8 output.
void launch_first_conv_cp8(const void* chunk, int in_dtype, Int3 chunk_size, const PatchPos* patches, int nb,
                           Int3 patch, const FirstConvW& w, __half* out, int parts, cudaStream_t s);
// Same from already extracted fp32 patches (nb,1,Z,Y,X) (plugin level / debug).
void launch_first_conv_cp8_from_patches(const float* patches, int nb, Int3 patch, const FirstConvW& w, __half* out,
                                        int parts, cudaStream_t s);

void launch_maxpool_cp8(const __half* in, __half* out, int channels, int parts, int nb, Int3 in_size, cudaStream_t s);
// ConvTranspose kernel=stride=(1,2,2), fp32 math on CUDA cores.  w: (cin, cout, 1,2,2) fp32.
void launch_convT_cp8(const __half* in, const float* w, const float* bias, __half* out, int cin, int cout,
                      int parts, int nb, Int3 in_size, cudaStream_t s);
// Fused network tail (reference patch/pytorch.py:105-113 + chunk/base.py:792-807): 1x1x1 head +
// sigmoid on the last CP8 activation, crop, x bump mask, accumulate into the output chunk with
// red.global.add -- the raw network output never touches HBM.
void launch_head_blend_cp8(const __half* in, const float* w, const float* bias, int cin, int cnet, int parts, Int3 in_patch,
                           Int3 out_patch, Int3 crop, const float* mask, const PatchPos* patches, int nb, float* out,
                           int channels, Int3 out_size, float scale, cudaStream_t s);

// 1x1x1 head + sigmoid -> planar fp32 (nb, cout, Z,Y,X).
void launch_head_sigmoid_cp8(const __half* in, const float* w, const float* bias, float* out, int cin, int cout,
                             int parts, int nb, Int3 size, cudaStream_t s);

}  // namespace cfb
