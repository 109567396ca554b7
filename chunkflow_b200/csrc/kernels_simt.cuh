// fp32 CUDA-core (FFMA) network kernels: the exact-fp32 precision mode and the device-side
// cross-check for the wgmma kernels.  Activations are planar (batch, C, Z, Y, X) fp32.
#pragma once
#include "common.cuh"

namespace cfb {

// 3x3x3 convolution, zero padding 1, optional ReLU.  The input is the channel
// concatenation [in0 (c0 channels), in1 (c1 channels)] (in1 may be null / c1 = 0).
// w: (cout, c0+c1, 3,3,3) fp32, bias: (cout).
void launch_conv3_f32(const float* in0, int c0, const float* in1, int c1, const float* w, const float* bias,
                      float* out, int cout, int nb, Int3 size, bool relu, cudaStream_t s);

// MaxPool (1,2,2).
void launch_maxpool_f32(const float* in, float* out, int channels, int nb, Int3 in_size, cudaStream_t s);

// ConvTranspose kernel=stride=(1,2,2): w (cin, cout, 1,2,2), bias (cout).  out is (nb,cout,Z,2Y,2X).
void launch_convT_f32(const float* in, const float* w, const float* bias, float* out, int cin, int cout,
                      int nb, Int3 in_size, cudaStream_t s);

// 1x1x1 convolution + sigmoid: w (cout, cin), bias (cout).
void launch_head_sigmoid_f32(const float* in, const float* w, const float* bias, float* out, int cin, int cout,
                             int nb, Int3 size, cudaStream_t s);

}  // namespace cfb
