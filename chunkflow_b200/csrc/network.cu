// Device-side 3-level U-Net: weight packing, workspace and layer dispatch.
#include "network.cuh"

#include <cstdlib>

#include "chunkflow_b200.h"
#include "kernels_memory.cuh"
#include "kernels_simt.cuh"

namespace cfb {

namespace {
struct Spec {
  const char* name;
  int cin, cout, taps;  // taps: 27 conv3, 4 convT, 1 head
};
// execution order; cout -1 = head (num channels from the weight tensor)
const Spec kSpecs[] = {
    {"enc0.0", 1, 16, 27},  {"enc0.2", 16, 16, 27}, {"enc1.0", 16, 32, 27}, {"enc1.2", 32, 32, 27},
    {"enc2.0", 32, 64, 27}, {"enc2.2", 64, 64, 27}, {"up1", 64, 32, 4},     {"dec1.0", 64, 32, 27},
    {"dec1.2", 32, 32, 27}, {"up0", 32, 16, 4},     {"dec0.0", 32, 16, 27}, {"dec0.2", 16, 16, 27},
    {"head", 16, -1, 1},
};
}  // namespace

void Network::configure(int precision, Int3 patch, int batch) {
  if (precision != CFB_PRECISION_F32_SIMT && precision != CFB_PRECISION_F16X3_UMMA && precision != CFB_PRECISION_F16_UMMA &&
      precision != CFB_PRECISION_F16F8_UMMA)
    throw std::invalid_argument("unknown precision mode");
  precision_ = precision;
  patch_ = patch;
  batch_ = batch;
}

void Network::release() {
  for (void* p : owned_) cudaFree(p);
  owned_.clear();
  for (auto& kv : layers_) { cudaFree(kv.second.w); cudaFree(kv.second.bias); free_packed(kv.second.packed); }
  layers_.clear();
  for (cudaEvent_t e : prof_pool_) cudaEventDestroy(e);
  prof_pool_.clear();
  ready_ = false;
  buf_in_ = nullptr;
  e0a_ = nullptr;
}

float* Network::patch_input_buffer(int nb) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  if (!buf_in_) {
    CFB_CUDA(cudaMalloc(&buf_in_, (size_t)vol(patch_) * batch_ * sizeof(float)));
    owned_.push_back(buf_in_);
  }
  return buf_in_;
}

void Network::allocate() {
  if (e0a_) return;
  const int64_t v0 = vol(patch_), v1 = v0 / 4, v2 = v0 / 16;
  auto alloc = [&](int64_t floats) {
    float* p = nullptr;
    CFB_CUDA(cudaMalloc(&p, (size_t)floats * batch_ * sizeof(float)));
    owned_.push_back(p);
    return p;
  };
  patch_input_buffer(1);
  net_out_ = alloc((int64_t)std::max(cnet_, 1) * v0);
  if (umma()) {
    const int P = parts();
    auto halloc = [&](int64_t channels, int64_t v) {
      __half* p = nullptr;
      CFB_CUDA(cudaMalloc(&p, (size_t)channels * P * v * batch_ * sizeof(__half)));
      owned_.push_back(p);
      return p;
    };
    h_e0a_ = halloc(16, v0); h_e0_ = halloc(16, v0); h_p0_ = halloc(16, v1);
    h_e1a_ = halloc(32, v1); h_e1_ = halloc(32, v1); h_p1_ = halloc(32, v2);
    h_e2a_ = halloc(64, v2); h_e2_ = halloc(64, v2);
    h_u1_ = halloc(32, v1); h_d1a_ = halloc(32, v1); h_d1_ = halloc(32, v1);
    h_u0_ = halloc(16, v0); h_d0a_ = halloc(16, v0); h_d0_ = halloc(16, v0);
    e0a_ = net_out_;  // marks "allocated"
    return;
  }
  e0a_ = alloc(16 * v0); e0_ = alloc(16 * v0); p0_ = alloc(16 * v1);
  e1a_ = alloc(32 * v1); e1_ = alloc(32 * v1); p1_ = alloc(32 * v2);
  e2a_ = alloc(64 * v2); e2_ = alloc(64 * v2);
  u1_ = alloc(32 * v1); d1a_ = alloc(32 * v1); d1_ = alloc(32 * v1);
  u0_ = alloc(16 * v0); d0a_ = alloc(16 * v0); d0_ = alloc(16 * v0);
}

bool Network::load(const std::map<std::string, std::vector<float>>& host_w, int num_output_channels, std::string& err) {
  ready_ = false;
  for (auto& kv : layers_) { cudaFree(kv.second.w); cudaFree(kv.second.bias); free_packed(kv.second.packed); }
  layers_.clear();
  for (const Spec& sp : kSpecs) {
    const std::string wn = std::string(sp.name) + ".weight", bn = std::string(sp.name) + ".bias";
    auto wi = host_w.find(wn), bi = host_w.find(bn);
    if (wi == host_w.end() || bi == host_w.end()) { err = "missing tensor " + (wi == host_w.end() ? wn : bn); return false; }
    int cout = sp.cout;
    if (cout < 0) {
      if (wi->second.size() % sp.cin) { err = "head.weight has a wrong size"; return false; }
      cout = (int)(wi->second.size() / sp.cin);
      cnet_ = cout;
    }
    if ((int64_t)wi->second.size() != (int64_t)sp.cin * cout * sp.taps) { err = wn + " has a wrong size"; return false; }
    if ((int)bi->second.size() != cout) { err = bn + " has a wrong size"; return false; }
    ConvLayer L;
    L.name = sp.name; L.cin = sp.cin; L.cout = cout;
    CFB_CUDA(cudaMalloc(&L.w, wi->second.size() * sizeof(float)));
    CFB_CUDA(cudaMalloc(&L.bias, bi->second.size() * sizeof(float)));
    CFB_CUDA(cudaMemcpy(L.w, wi->second.data(), wi->second.size() * sizeof(float), cudaMemcpyHostToDevice));
    CFB_CUDA(cudaMemcpy(L.bias, bi->second.data(), bi->second.size() * sizeof(float), cudaMemcpyHostToDevice));
    if (umma() && sp.taps == 27 && sp.cin >= 16)
      pack_conv3_weights(wi->second.data(), bi->second.data(), sp.cin, cout, fmt(), L.packed);
    if (umma() && sp.taps == 4)
      pack_convT_weights(wi->second.data(), bi->second.data(), sp.cin, cout, fmt(), L.packed);
    if (umma() && sp.taps == 27 && sp.cin == 1 && cout == 16) {
      for (int t = 0; t < 27; ++t)
        for (int c = 0; c < 16; ++c) first_w_.w[t][c] = wi->second[(size_t)c * 27 + t];
      for (int c = 0; c < 16; ++c) first_w_.b[c] = bi->second[c];
    }
    layers_[sp.name] = L;
  }
  if (num_output_channels > cnet_) { err = "the network produces fewer channels than num_output_channels"; return false; }
  if (cnet_ > 8) { err = "at most 8 network output channels are supported"; return false; }
  allocate();
  ready_ = true;
  return true;
}

void Network::set_profiling(bool on) {
  profiling_ = on;
  std::vector<std::string> n; std::vector<float> m; std::vector<int64_t> l;
  layer_timing(n, m, l);  // drain
  prof_names_.clear(); prof_ms_.clear(); prof_launches_.clear();
}

void Network::prof_begin(const char* name, cudaStream_t s) {
  if (!profiling_) return;
  int id = -1;
  for (size_t i = 0; i < prof_names_.size(); ++i) if (prof_names_[i] == name) id = (int)i;
  if (id < 0) { id = (int)prof_names_.size(); prof_names_.push_back(name); prof_ms_.push_back(0.f); prof_launches_.push_back(0); }
  auto get = [&]() {
    cudaEvent_t e;
    if (!prof_pool_.empty()) { e = prof_pool_.back(); prof_pool_.pop_back(); } else { CFB_CUDA(cudaEventCreate(&e)); }
    return e;
  };
  Span sp{id, get(), get()};
  CFB_CUDA(cudaEventRecord(sp.a, s));
  prof_spans_.push_back(sp);
  prof_cur_ = (int)prof_spans_.size() - 1;
}

void Network::prof_end(cudaStream_t s) {
  if (!profiling_ || prof_cur_ < 0) return;
  CFB_CUDA(cudaEventRecord(prof_spans_[prof_cur_].b, s));
  prof_cur_ = -1;
}

void Network::layer_timing(std::vector<std::string>& names, std::vector<float>& ms, std::vector<int64_t>& launches) {
  for (Span& sp : prof_spans_) {
    CFB_CUDA(cudaEventSynchronize(sp.b));
    float t = 0.f;
    CFB_CUDA(cudaEventElapsedTime(&t, sp.a, sp.b));
    prof_ms_[sp.id] += t;
    prof_launches_[sp.id] += 1;
    prof_pool_.push_back(sp.a);
    prof_pool_.push_back(sp.b);
  }
  prof_spans_.clear();
  names = prof_names_; ms = prof_ms_; launches = prof_launches_;
}

int Network::forward(int nb, cudaStream_t s) {
  const Int3 s0 = patch_, s1{patch_.z, patch_.y / 2, patch_.x / 2}, s2{patch_.z, patch_.y / 4, patch_.x / 4};
  auto conv = [&](const char* name, const float* a, int ca, const float* b, int cb, float* out, Int3 sz) {
    const ConvLayer& L = layers_.at(name);
    prof_begin(name, s);
    launch_conv3_f32(a, ca, b, cb, L.w, L.bias, out, L.cout, nb, sz, /*relu=*/true, s);
    prof_end(s);
  };
  conv("enc0.0", buf_in_, 1, nullptr, 0, e0a_, s0);
  conv("enc0.2", e0a_, 16, nullptr, 0, e0_, s0);
  prof_begin("pool0", s); launch_maxpool_f32(e0_, p0_, 16, nb, s0, s); prof_end(s);
  conv("enc1.0", p0_, 16, nullptr, 0, e1a_, s1);
  conv("enc1.2", e1a_, 32, nullptr, 0, e1_, s1);
  prof_begin("pool1", s); launch_maxpool_f32(e1_, p1_, 32, nb, s1, s); prof_end(s);
  conv("enc2.0", p1_, 32, nullptr, 0, e2a_, s2);
  conv("enc2.2", e2a_, 64, nullptr, 0, e2_, s2);
  { const ConvLayer& L = layers_.at("up1"); prof_begin("up1", s); launch_convT_f32(e2_, L.w, L.bias, u1_, 64, 32, nb, s2, s); prof_end(s); }
  conv("dec1.0", u1_, 32, e1_, 32, d1a_, s1);  // torch.cat([up1, enc1])
  conv("dec1.2", d1a_, 32, nullptr, 0, d1_, s1);
  { const ConvLayer& L = layers_.at("up0"); prof_begin("up0", s); launch_convT_f32(d1_, L.w, L.bias, u0_, 32, 16, nb, s1, s); prof_end(s); }
  conv("dec0.0", u0_, 16, e0_, 16, d0a_, s0);  // torch.cat([up0, enc0])
  conv("dec0.2", d0a_, 16, nullptr, 0, d0_, s0);
  { const ConvLayer& L = layers_.at("head"); prof_begin("head", s); launch_head_sigmoid_f32(d0_, L.w, L.bias, net_out_, 16, cnet_, nb, s0, s); prof_end(s); }
  return 15;
}

int Network::forward_cp8(const void* chunk, int in_dtype, Int3 cs, const PatchPos* patches, int nb, cudaStream_t s,
                         bool with_head, const ConvTail* tail) {
  const Int3 s0 = patch_, s1{patch_.z, patch_.y / 2, patch_.x / 2}, s2{patch_.z, patch_.y / 4, patch_.x / 4};
  const int P = fmt();  // the CUDA-core CP8 kernels take the number format
  {
    const ConvLayer& L = layers_.at("enc0.0");
    prof_begin("enc0.0", s);
    if (chunk) launch_first_conv_cp8(chunk, in_dtype, cs, patches, nb, s0, L.w, L.bias, h_e0a_, P, s,
                                     getenv("CFB_FIRST_CONV_SMEM_W") ? nullptr : &first_w_);
    else launch_first_conv_cp8_from_patches(buf_in_, nb, s0, L.w, L.bias, h_e0a_, P, s);
    prof_end(s);
  }
  auto conv = [&](const char* name, const __half* a, int ca, const __half* b, int cb, __half* out, Int3 sz, __half* pool_out = nullptr) {
    const ConvLayer& L = layers_.at(name);
    prof_begin(name, s);
    launch_conv3_wgmma(a, ca, b, cb, L.packed, out, nb, sz, /*relu=*/true, s, nullptr, pool_out);
    prof_end(s);
  };
  // the two encoder outputs feed a (1,2,2) max pool: fused into the convolution's epilogue unless CFB_NO_POOL_FUSION is set
  const bool fuse_pool = getenv("CFB_NO_POOL_FUSION") == nullptr;
  int launches_saved = 0;
  conv("enc0.2", h_e0a_, 16, nullptr, 0, h_e0_, s0, fuse_pool ? h_p0_ : nullptr);
  if (!fuse_pool) { prof_begin("pool0", s); launch_maxpool_cp8(h_e0_, h_p0_, 16, P, nb, s0, s); prof_end(s); } else ++launches_saved;
  conv("enc1.0", h_p0_, 16, nullptr, 0, h_e1a_, s1);
  conv("enc1.2", h_e1a_, 32, nullptr, 0, h_e1_, s1, fuse_pool ? h_p1_ : nullptr);
  if (!fuse_pool) { prof_begin("pool1", s); launch_maxpool_cp8(h_e1_, h_p1_, 32, P, nb, s1, s); prof_end(s); } else ++launches_saved;
  conv("enc2.0", h_p1_, 32, nullptr, 0, h_e2a_, s2);
  conv("enc2.2", h_e2a_, 64, nullptr, 0, h_e2_, s2);
  // transposed convolutions on wgmma; CFB_SIMT_CONVT selects the CUDA-core kernel (fp32 math, a cross-check)
  const bool simt_up = getenv("CFB_SIMT_CONVT") != nullptr;
  { const ConvLayer& L = layers_.at("up1"); prof_begin("up1", s);
    if (simt_up) launch_convT_cp8(h_e2_, L.w, L.bias, h_u1_, 64, 32, P, nb, s2, s); else launch_convT_wgmma(h_e2_, L.packed, h_u1_, nb, s2, s);
    prof_end(s); }
  conv("dec1.0", h_u1_, 32, h_e1_, 32, h_d1a_, s1);  // torch.cat([up1, enc1])
  conv("dec1.2", h_d1a_, 32, nullptr, 0, h_d1_, s1);
  { const ConvLayer& L = layers_.at("up0"); prof_begin("up0", s);
    if (simt_up) launch_convT_cp8(h_d1_, L.w, L.bias, h_u0_, 32, 16, P, nb, s1, s); else launch_convT_wgmma(h_d1_, L.packed, h_u0_, nb, s1, s);
    prof_end(s); }
  conv("dec0.0", h_u0_, 16, h_e0_, 16, h_d0a_, s0);  // torch.cat([up0, enc0])
  if (tail) {  // 3x3x3 conv + ReLU + 1x1x1 head + sigmoid + crop + bump mask + blend in one kernel
    const ConvLayer& L = layers_.at("dec0.2");
    prof_begin("dec0.2+head+blend", s);
    launch_conv3_wgmma(h_d0a_, 16, nullptr, 0, L.packed, h_d0_, nb, s0, /*relu=*/true, s, tail);
    prof_end(s);
    return 14 - launches_saved;
  }
  conv("dec0.2", h_d0a_, 16, nullptr, 0, h_d0_, s0);
  if (!with_head) return 14 - launches_saved;  // the head is fused into the blend kernel
  { const ConvLayer& L = layers_.at("head"); prof_begin("head", s); launch_head_sigmoid_cp8(h_d0_, L.w, L.bias, net_out_, 16, cnet_, P, nb, s0, s); prof_end(s); }
  return 15 - launches_saved;
}

int Network::forward_from_chunk(const void* chunk, int in_dtype, Int3 cs, const PatchPos* patches, int nb, cudaStream_t s) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  if (umma()) return forward_cp8(chunk, in_dtype, cs, patches, nb, s, /*with_head=*/false);
  prof_begin("extract", s);
  launch_extract_patches(chunk, in_dtype, cs, patches, nb, patch_, buf_in_, s);
  prof_end(s);
  return 1 + forward(nb, s);
}

int Network::forward_and_blend(const void* chunk, int in_dtype, Int3 cs, const PatchPos* patches, int nb, Int3 op, Int3 crop,
                               const float* mask, float* out, int channels, Int3 out_size, float scale, cudaStream_t s) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  if (umma() && !getenv("CFB_NO_FUSED_TAIL")) {
    const ConvLayer& H = layers_.at("head");
    ConvTail tail{H.w, H.bias, patches, mask, out, channels, op, crop, out_size, scale};
    return forward_cp8(chunk, in_dtype, cs, patches, nb, s, /*with_head=*/false, &tail);
  }
  int n = forward_from_chunk(chunk, in_dtype, cs, patches, nb, s);
  return n + blend(op, crop, mask, patches, nb, out, channels, out_size, scale, s);
}

int Network::forward_from_host_patches(const float* h_patches, int nb, cudaStream_t s) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  CFB_CUDA(cudaMemcpyAsync(buf_in_, h_patches, (size_t)nb * vol(patch_) * sizeof(float), cudaMemcpyHostToDevice, s));
  if (umma()) return forward_cp8(nullptr, 0, Int3{0, 0, 0}, nullptr, nb, s, /*with_head=*/true);
  return forward(nb, s);
}

int Network::blend(Int3 op, Int3 crop, const float* mask, const PatchPos* patches, int nb, float* out, int channels,
                   Int3 out_size, float scale, cudaStream_t s) {
  if (umma()) {
    const ConvLayer& L = layers_.at("head");
    prof_begin("head+blend", s);
    launch_head_blend_cp8(h_d0_, L.w, L.bias, 16, cnet_, fmt(), patch_, op, crop, mask, patches, nb, out, channels, out_size, scale, s);
    prof_end(s);
    return 1;
  }
  prof_begin("blend", s);
  launch_blend_patches(net_out_, cnet_, patch_, op, crop, mask, patches, nb, out, channels, out_size, scale, s);
  prof_end(s);
  return 1;
}

void Network::crop_mask(Int3 op, Int3 crop, const float* mask, int nb, float* dst, int channels, cudaStream_t s) {
  launch_crop_mask(net_out_, cnet_, patch_, op, crop, mask, nb, dst, channels, /*repeat=*/false, s);
}

void Network::copy_raw_output_to_host(float* h_out, cudaStream_t s) {
  CFB_CUDA(cudaMemcpyAsync(h_out, net_out_, (size_t)cnet_ * vol(patch_) * sizeof(float), cudaMemcpyDeviceToHost, s));
}

int Network::debug_conv3(const float* h_in, int cin, Int3 size, const float* h_w, const float* h_b, int cout, bool relu,
                         float* h_out, cudaStream_t s) {
  float *d_in = nullptr, *d_w = nullptr, *d_b = nullptr, *d_out = nullptr;
  const int64_t v = vol(size);
  CFB_CUDA(cudaMalloc(&d_in, (size_t)cin * v * 4));
  CFB_CUDA(cudaMalloc(&d_w, (size_t)cout * cin * 27 * 4));
  CFB_CUDA(cudaMalloc(&d_b, (size_t)cout * 4));
  CFB_CUDA(cudaMalloc(&d_out, (size_t)cout * v * 4));
  CFB_CUDA(cudaMemcpyAsync(d_in, h_in, (size_t)cin * v * 4, cudaMemcpyHostToDevice, s));
  CFB_CUDA(cudaMemcpyAsync(d_w, h_w, (size_t)cout * cin * 27 * 4, cudaMemcpyHostToDevice, s));
  CFB_CUDA(cudaMemcpyAsync(d_b, h_b, (size_t)cout * 4, cudaMemcpyHostToDevice, s));
  if (umma()) {
    if (cin % 16) { cudaFree(d_in); cudaFree(d_w); cudaFree(d_b); cudaFree(d_out); throw std::runtime_error("the wgmma convolution needs cin % 16 == 0"); }
    const int P = parts();
    __half *c_in = nullptr, *c_out = nullptr;
    CFB_CUDA(cudaMalloc(&c_in, (size_t)cin * P * v * 2));
    CFB_CUDA(cudaMalloc(&c_out, (size_t)cout * P * v * 2));
    PackedConv pk;
    pack_conv3_weights(h_w, h_b, cin, cout, fmt(), pk);
    launch_planar_to_cp8(d_in, c_in, cin, fmt(), 1, size, s);
    // exercise the two-source (concat) path whenever the channel count allows it
    const int ca = cin >= 32 ? cin / 2 : cin, cb = cin - ca;
    launch_conv3_wgmma(c_in, ca, cb ? c_in + (size_t)ca * P * v : nullptr, cb, pk, c_out, 1, size, relu, s);
    launch_cp8_to_planar(c_out, d_out, cout, fmt(), 1, size, s);
    CFB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)cout * v * 4, cudaMemcpyDeviceToHost, s));
    cudaError_t err = cudaStreamSynchronize(s);
    cudaFree(c_in); cudaFree(c_out); free_packed(pk);
    cudaFree(d_in); cudaFree(d_w); cudaFree(d_b); cudaFree(d_out);
    CFB_CUDA(err);
    return CFB_OK;
  }
  launch_conv3_f32(d_in, cin, nullptr, 0, d_w, d_b, d_out, cout, 1, size, relu, s);
  CFB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)cout * v * 4, cudaMemcpyDeviceToHost, s));
  CFB_CUDA(cudaStreamSynchronize(s));
  cudaFree(d_in); cudaFree(d_w); cudaFree(d_b); cudaFree(d_out);
  return CFB_OK;
}

}  // namespace cfb
