// The fixed 3-level 3D U-Net (chunkflow_b200/convnet/unet3l.py) on the device.
// Owns the packed weights and the activation workspace for `batch` patches in flight and
// dispatches each layer to the kernels of the configured precision mode.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels_conv.cuh"

namespace cfb {

struct ConvLayer {
  std::string name;
  int cin = 0, cout = 0;
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

  // Extract `nb` patches from the chunk and run the network; returns kernel launches.
  int forward_from_chunk(const void* chunk, int in_dtype, Int3 chunk_size, const PatchPos* patches, int nb,
                         cudaStream_t s);
  int forward_from_host_patches(const float* h_patches, int nb, cudaStream_t s);
  // Whole-chunk path: extract + network + crop + bump mask + accumulate into the output chunk.  On the wgmma
  // path the head and the blend are fused into the epilogue of the last convolution.
  int forward_and_blend(const void* chunk, int in_dtype, Int3 chunk_size, const PatchPos* patches, int nb, Int3 out_patch,
                        Int3 crop, const float* mask, float* out, int channels, Int3 out_size, float scale, cudaStream_t s);
  // crop + bump mask + accumulate the last forward's outputs into the output chunk.
  int blend(Int3 out_patch, Int3 crop, const float* mask, const PatchPos* patches, int nb, float* out,
            int channels, Int3 out_size, float scale, cudaStream_t s);
  void crop_mask(Int3 out_patch, Int3 crop, const float* mask, int nb, float* dst, int channels, cudaStream_t s);
  float* patch_input_buffer(int nb);
  void copy_raw_output_to_host(float* h_out, cudaStream_t s);
  // per-layer CUDA-event profiling
  void set_profiling(bool on);
  void layer_timing(std::vector<std::string>& names, std::vector<float>& ms, std::vector<int64_t>& launches);

  int debug_conv3(const float* h_in, int cin, Int3 size, const float* h_w, const float* h_b, int cout, bool relu,
                  float* h_out, cudaStream_t s);

 private:
  void allocate();
  int forward(int nb, cudaStream_t s);  // from buf_in_ (fp32 SIMT path)
  // wgmma path: chunk != nullptr -> first layer reads the chunk, else the staged fp32 patches in buf_in_
  int forward_cp8(const void* chunk, int in_dtype, Int3 chunk_size, const PatchPos* patches, int nb, cudaStream_t s,
                  bool with_head, const ConvTail* tail = nullptr);
  bool umma() const { return precision_ != 0; }
  // activation number format of the wgmma path (act_format.cuh) and its planes per 8-channel chunk
  int fmt() const { return precision_ == 1 ? kFmtF16x2 : (precision_ == 3 ? kFmtF16F8 : kFmtF16); }
  int parts() const { return fmt_planes(fmt()); }

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
  FirstConvW first_w_{};  // host copy of the first layer, passed to its kernel by value
  std::map<std::string, ConvLayer> layers_;
  std::vector<void*> owned_;
  // fp32 planar activations, (batch, C, Z, Y, X)
  float *buf_in_ = nullptr, *e0a_ = nullptr, *e0_ = nullptr, *p0_ = nullptr, *e1a_ = nullptr, *e1_ = nullptr,
        *p1_ = nullptr, *e2a_ = nullptr, *e2_ = nullptr, *u1_ = nullptr, *d1a_ = nullptr, *d1_ = nullptr,
        *u0_ = nullptr, *d0a_ = nullptr, *d0_ = nullptr, *net_out_ = nullptr;
  // CP8 fp16 activations of the wgmma path
  __half *h_e0a_ = nullptr, *h_e0_ = nullptr, *h_p0_ = nullptr, *h_e1a_ = nullptr, *h_e1_ = nullptr, *h_p1_ = nullptr,
         *h_e2a_ = nullptr, *h_e2_ = nullptr, *h_u1_ = nullptr, *h_d1a_ = nullptr, *h_d1_ = nullptr, *h_u0_ = nullptr,
         *h_d0a_ = nullptr, *h_d0_ = nullptr;
};

}  // namespace cfb
