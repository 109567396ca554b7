// The plain 3D U-Net family of chunkflow_b200/convnet/unet3l.py (depth 2, 3 or 4, widths 16, 32, ..., (1,2,2) pooling) on
// the device.  The layer table is generated from the depth and widths found in the state dict; the network owns the packed
// weights and the activation workspace for `batch` patches in flight and dispatches each layer to the kernels of the
// configured precision mode.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"
#include "kernels_conv.cuh"

namespace cfb {

// Activations are numbered by the layer table (network.cu); the input patches and the raw output come first.
using Act = int;
constexpr Act kIn = 0, kOut = 1, kNoAct = -1;

struct ConvLayer {
  float* w = nullptr;     // fp32, state_dict layout
  float* bias = nullptr;  // fp32
  PackedConv packed;      // B-operand blocks for the wgmma path (3x3x3 layers, cin >= 16)
};

class Network {
 public:
  void configure(int precision, Int3 patch, int batch);
  bool load(const std::map<std::string, std::vector<float>>& host_w, int num_output_channels, std::string& err);
  bool ready() const { return ready_; }
  int cnet() const { return cnet_; }
  void release();

  // Whole-chunk path: extract + network + crop + bump mask + accumulate into the output chunk; returns kernel launches.
  // On the tensor-core path the head and the blend are fused into the epilogue of the last convolution.
  int forward_and_blend(const void* chunk, int in_dtype, Int3 chunk_size, const PatchPos* patches, int nb, Int3 out_patch,
                        Int3 crop, const float* mask, float* out, int channels, Int3 out_size, float scale, cudaStream_t s);
  // Network on `nb` fp32 patches from the host; the raw output stays on the device (crop_mask, copy_raw_output_to_host).
  int forward_from_host_patches(const float* h_patches, int nb, cudaStream_t s);
  void crop_mask(Int3 out_patch, Int3 crop, const float* mask, int nb, float* dst, int channels, cudaStream_t s);
  float* patch_input_buffer(int nb);
  void copy_raw_output_to_host(float* h_out, cudaStream_t s);
  // per-layer CUDA-event profiling
  void set_profiling(bool on);
  void layer_timing(std::vector<std::string>& names, std::vector<float>& ms, std::vector<int64_t>& launches);

  // One step of the layer table on host arrays (cfb_debug_layer_host); the network's own weights and workspace are not used.
  int debug_layer(const cfb_layer_args& a, cudaStream_t s);

 private:
  // How the network ends: head + blend in the epilogue of the last convolution, head + blend (tensor cores: one CUDA-core
  // kernel, simt: the head, then the blend kernel), or the head into the raw output.
  enum End { kFusedTail, kBlend, kRawOutput };
  // Environment switches, read once per forward call, that route it through kernels which cross-check the production ones.
  struct CrossChecks {
    bool no_pool_fusion;  // CFB_NO_POOL_FUSION: the (1,2,2) max pools as kernels of their own
    bool simt_convt;      // CFB_SIMT_CONVT: the transposed convolutions on CUDA cores
    bool no_fused_tail;   // CFB_NO_FUSED_TAIL: the head + blend as a kernel of its own
  };
  static CrossChecks read_cross_checks();
  struct Route {
    const void* chunk;  // the first layer reads the patches blend.patches from this chunk, or (nullptr) the staged fp32 patches
    int in_dtype;
    Int3 chunk_size;
    End end;
    ConvTail blend;     // the output of the blending ends; run fills in the head
    CrossChecks checks;
  };
  // Issues every step of the layer table for `nb` patches with the kernels of the configured mode; returns the launches.
  int run(const Route& r, int nb, cudaStream_t s);

  enum Op { kOpFirst, kOpConv3, kOpConv3Pool, kOpConvT, kOpHead };
  struct Step {
    std::string name;  // profiling name; "<name>.weight" and "<name>.bias" in the state dict
    Op op;             // kOpFirst: 3x3x3 conv from the input patches; kOpConv3Pool: 3x3x3 conv feeding a (1,2,2) max pool
    int cin, cout;     // cout -1: the head, whose channels come from its weight tensor
    Act a, b;          // source, and the skip connection concatenated after it (torch.cat([a, b]))
    Act dst, pool;     // output, and its (1,2,2) max pool
    int level;         // resolution of the sources: (Y, X) >> level
  };
  // The layer table of the U-Net of this depth and widths (16 << level), in execution order; `acts` gets the activation count.
  static std::vector<Step> make_steps(int depth, int& acts);
  static int taps(Op op);
  int act_channels(Act a) const;
  void allocate();
  bool tensor_cores() const { return precision_ != CFB_PRECISION_F32_SIMT; }
  // activation number format of the tensor-core path (act_format.cuh) and its planes per 8-channel chunk
  int fmt() const {
    return precision_ == CFB_PRECISION_F16X3_UMMA ? kFmtF16x2 : precision_ == CFB_PRECISION_F16F8_UMMA ? kFmtF16F8 : kFmtF16;
  }
  int parts() const { return fmt_planes(fmt()); }
  float* f32(Act a) const { return act_[a].as<float>(); }
  __half* cp8(Act a) const { return act_[a].as<__half>(); }

  struct Span { int id; cudaEvent_t a, b; };
  void prof_begin(const char* name, cudaStream_t s);
  void prof_end(cudaStream_t s);
  bool profiling_ = false;
  std::vector<std::string> prof_names_;
  std::vector<float> prof_ms_;
  std::vector<int64_t> prof_launches_;
  std::vector<Span> prof_spans_;
  std::vector<cudaEvent_t> prof_pool_;
  int prof_cur_ = -1;

  int precision_ = 0;
  Int3 patch_{0, 0, 0};
  int batch_ = 1;
  bool ready_ = false;
  int cnet_ = 0;
  FirstConvW first_w_{};              // host copy of the first layer, passed to its kernel by value
  int depth_ = 0;                     // levels of the committed network, 0 before the first commit
  std::vector<Step> steps_;           // the layer table of the committed network
  std::vector<ConvLayer> layers_;     // by index into the layer table
  // (batch, C, Z, Y, X) fp32 for kIn, kOut and every activation of the simt mode, CP8 for the tensor-core modes
  std::vector<DeviceBuffer> act_ = std::vector<DeviceBuffer>(2);
};

}  // namespace cfb
