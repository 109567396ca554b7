// Device-side 3-level U-Net: weight packing, workspace and layer dispatch.
#include "network.cuh"

#include <cstdlib>

#include "chunkflow_b200.h"
#include "kernels_memory.cuh"
#include "kernels_simt.cuh"

namespace cfb {

namespace {
enum Op { kOpFirst, kOpConv3, kOpConv3Pool, kOpConvT, kOpHead };
struct Step {
  const char* name;  // profiling name; "<name>.weight" and "<name>.bias" in the state dict
  Op op;             // kOpFirst: 3x3x3 conv from the input patches; kOpConv3Pool: 3x3x3 conv feeding a (1,2,2) max pool
  int cin, cout;     // cout -1: the head, whose channels come from its weight tensor
  Act a, b;          // source, and the skip connection concatenated after it (torch.cat([a, b]))
  Act dst, pool;     // output, and its (1,2,2) max pool
  int level;         // resolution of the sources: the patch, then (Y/2, X/2) and (Y/4, X/4)
};
// execution order
const Step kNet[] = {
    {"enc0.0", kOpFirst, 1, 16, kIn, kNoAct, kE0a, kNoAct, 0},
    {"enc0.2", kOpConv3Pool, 16, 16, kE0a, kNoAct, kE0, kP0, 0},
    {"enc1.0", kOpConv3, 16, 32, kP0, kNoAct, kE1a, kNoAct, 1},
    {"enc1.2", kOpConv3Pool, 32, 32, kE1a, kNoAct, kE1, kP1, 1},
    {"enc2.0", kOpConv3, 32, 64, kP1, kNoAct, kE2a, kNoAct, 2},
    {"enc2.2", kOpConv3, 64, 64, kE2a, kNoAct, kE2, kNoAct, 2},
    {"up1", kOpConvT, 64, 32, kE2, kNoAct, kU1, kNoAct, 2},
    {"dec1.0", kOpConv3, 64, 32, kU1, kE1, kD1a, kNoAct, 1},
    {"dec1.2", kOpConv3, 32, 32, kD1a, kNoAct, kD1, kNoAct, 1},
    {"up0", kOpConvT, 32, 16, kD1, kNoAct, kU0, kNoAct, 1},
    {"dec0.0", kOpConv3, 32, 16, kU0, kE0, kD0a, kNoAct, 0},
    {"dec0.2", kOpConv3, 16, 16, kD0a, kNoAct, kD0, kNoAct, 0},
    {"head", kOpHead, 16, -1, kD0, kNoAct, kOut, kNoAct, 0},
};
constexpr int kSteps = sizeof(kNet) / sizeof(kNet[0]);
const char* const kPoolName[] = {"pool0", "pool1"};  // by level

int taps(Op op) { return op == kOpConvT ? 4 : op == kOpHead ? 1 : 27; }
// channels of an activation: the input patches have one, every other one those of the step that produces it
int act_channels(Act a) {
  for (const Step& st : kNet)
    if (st.dst == a || st.pool == a) return st.cout;
  return 1;
}
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
  for (ConvLayer& L : layers_) { cudaFree(L.w); cudaFree(L.bias); free_packed(L.packed); }
  layers_.clear();
  for (cudaEvent_t e : prof_pool_) cudaEventDestroy(e);
  prof_pool_.clear();
  ready_ = false;
  act_.fill(nullptr);
}

float* Network::patch_input_buffer(int nb) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  if (!act_[kIn]) {
    CFB_CUDA(cudaMalloc(&act_[kIn], (size_t)vol(patch_) * batch_ * sizeof(float)));
    owned_.push_back(act_[kIn]);
  }
  return f32(kIn);
}

void Network::allocate() {
  if (act_[kOut]) return;
  patch_input_buffer(1);
  auto alloc = [&](Act a, size_t bytes_per_voxel, int level) {
    CFB_CUDA(cudaMalloc(&act_[a], bytes_per_voxel * (size_t)(vol(patch_) >> (2 * level)) * batch_));
    owned_.push_back(act_[a]);
  };
  alloc(kOut, sizeof(float) * std::max(cnet_, 1), 0);
  const size_t bytes = tensor_cores() ? sizeof(__half) * parts() : sizeof(float);  // per channel and voxel
  for (const Step& st : kNet) {
    if (st.op == kOpHead) continue;
    alloc(st.dst, bytes * st.cout, st.op == kOpConvT ? st.level - 1 : st.level);
    if (st.pool != kNoAct) alloc(st.pool, bytes * st.cout, st.level + 1);
  }
}

bool Network::load(const std::map<std::string, std::vector<float>>& host_w, int num_output_channels, std::string& err) {
  ready_ = false;
  for (ConvLayer& L : layers_) { cudaFree(L.w); cudaFree(L.bias); free_packed(L.packed); }
  layers_.clear();
  for (const Step& st : kNet) {
    const std::string wn = std::string(st.name) + ".weight", bn = std::string(st.name) + ".bias";
    auto wi = host_w.find(wn), bi = host_w.find(bn);
    if (wi == host_w.end() || bi == host_w.end()) { err = "missing tensor " + (wi == host_w.end() ? wn : bn); return false; }
    const std::vector<float>& w = wi->second;
    const std::vector<float>& b = bi->second;
    int cout = st.cout;
    if (st.op == kOpHead) {
      if (w.size() % st.cin) { err = "head.weight has a wrong size"; return false; }
      cout = (int)(w.size() / st.cin);
      cnet_ = cout;
    }
    if ((int64_t)w.size() != (int64_t)st.cin * cout * taps(st.op)) { err = wn + " has a wrong size"; return false; }
    if ((int)b.size() != cout) { err = bn + " has a wrong size"; return false; }
    ConvLayer L;
    CFB_CUDA(cudaMalloc(&L.w, w.size() * sizeof(float)));
    CFB_CUDA(cudaMalloc(&L.bias, b.size() * sizeof(float)));
    CFB_CUDA(cudaMemcpy(L.w, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice));
    CFB_CUDA(cudaMemcpy(L.bias, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice));
    if (tensor_cores() && (st.op == kOpConv3 || st.op == kOpConv3Pool))
      pack_conv3_weights(w.data(), b.data(), st.cin, cout, fmt(), L.packed);
    if (tensor_cores() && st.op == kOpConvT) pack_convT_weights(w.data(), b.data(), st.cin, cout, fmt(), L.packed);
    if (tensor_cores() && st.op == kOpFirst) {
      for (int t = 0; t < 27; ++t)
        for (int c = 0; c < 16; ++c) first_w_.w[t][c] = w[(size_t)c * 27 + t];
      for (int c = 0; c < 16; ++c) first_w_.b[c] = b[c];
    }
    layers_.push_back(L);
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

Network::CrossChecks Network::read_cross_checks() {
  return {getenv("CFB_NO_POOL_FUSION") != nullptr, getenv("CFB_SIMT_CONVT") != nullptr, getenv("CFB_NO_FUSED_TAIL") != nullptr};
}

int Network::run(const Route& r, int nb, cudaStream_t s) {
  const bool tc = tensor_cores();
  const int P = fmt();  // the CUDA-core CP8 kernels take the number format
  ConvTail blend = r.blend;
  blend.head_w = layers_[kSteps - 1].w;
  blend.head_b = layers_[kSteps - 1].bias;
  int launches = 0;
  auto issue = [&](const char* name, auto&& launch) {
    prof_begin(name, s);
    launch();
    prof_end(s);
    ++launches;
  };
  for (int i = 0; i < kSteps; ++i) {
    const Step& st = kNet[i];
    const ConvLayer& L = layers_[i];
    const Int3 sz{patch_.z, patch_.y >> st.level, patch_.x >> st.level};
    const int cb = st.b == kNoAct ? 0 : act_channels(st.b), ca = st.cin - cb;
    if (st.op == kOpFirst) {
      if (!tc && r.chunk)
        issue("extract", [&] { launch_extract_patches(r.chunk, r.in_dtype, r.chunk_size, blend.patches, nb, patch_, f32(kIn), s); });
      issue(st.name, [&] {
        if (!tc) launch_conv3_f32(f32(kIn), 1, nullptr, 0, L.w, L.bias, f32(st.dst), st.cout, nb, sz, /*relu=*/true, s);
        else if (r.chunk) launch_first_conv_cp8(r.chunk, r.in_dtype, r.chunk_size, blend.patches, nb, sz, first_w_, cp8(st.dst), P, s);
        else launch_first_conv_cp8_from_patches(f32(kIn), nb, sz, first_w_, cp8(st.dst), P, s);
      });
    } else if (st.op == kOpConv3 || st.op == kOpConv3Pool) {
      const bool pool = st.op == kOpConv3Pool, fuse_pool = tc && pool && !r.checks.no_pool_fusion;
      const bool fuse_tail = r.end == kFusedTail && kNet[i + 1].op == kOpHead;  // + head + sigmoid + crop + mask + blend
      issue(fuse_tail ? (std::string(st.name) + "+head+blend").c_str() : st.name, [&] {
        if (!tc) launch_conv3_f32(f32(st.a), ca, cb ? f32(st.b) : nullptr, cb, L.w, L.bias, f32(st.dst), st.cout, nb, sz, true, s);
        else launch_conv3_wgmma(cp8(st.a), ca, cb ? cp8(st.b) : nullptr, cb, L.packed, cp8(st.dst), nb, sz, /*relu=*/true, s,
                                fuse_tail ? &blend : nullptr, fuse_pool ? cp8(st.pool) : nullptr);
      });
      if (pool && !fuse_pool)
        issue(kPoolName[st.level], [&] {
          if (tc) launch_maxpool_cp8(cp8(st.dst), cp8(st.pool), st.cout, P, nb, sz, s);
          else launch_maxpool_f32(f32(st.dst), f32(st.pool), st.cout, nb, sz, s);
        });
    } else if (st.op == kOpConvT) {
      issue(st.name, [&] {
        if (!tc) launch_convT_f32(f32(st.a), L.w, L.bias, f32(st.dst), st.cin, st.cout, nb, sz, s);
        else if (r.checks.simt_convt) launch_convT_cp8(cp8(st.a), L.w, L.bias, cp8(st.dst), st.cin, st.cout, P, nb, sz, s);
        else launch_convT_wgmma(cp8(st.a), L.packed, cp8(st.dst), nb, sz, s);
      });
    } else if (r.end == kBlend && tc) {
      issue("head+blend", [&] {
        launch_head_blend_cp8(cp8(st.a), L.w, L.bias, st.cin, cnet_, P, sz, blend.out_patch, blend.crop, blend.mask, blend.patches,
                              nb, blend.out, blend.channels, blend.out_size, blend.scale, s);
      });
    } else if (r.end != kFusedTail) {
      issue(st.name, [&] {
        if (tc) launch_head_sigmoid_cp8(cp8(st.a), L.w, L.bias, f32(st.dst), st.cin, cnet_, P, nb, sz, s);
        else launch_head_sigmoid_f32(f32(st.a), L.w, L.bias, f32(st.dst), st.cin, cnet_, nb, sz, s);
      });
      if (r.end == kBlend)
        issue("blend", [&] {
          launch_blend_patches(f32(st.dst), cnet_, patch_, blend.out_patch, blend.crop, blend.mask, blend.patches, nb, blend.out,
                               blend.channels, blend.out_size, blend.scale, s);
        });
    }
  }
  return launches;
}

int Network::forward_and_blend(const void* chunk, int in_dtype, Int3 cs, const PatchPos* patches, int nb, Int3 op, Int3 crop,
                               const float* mask, float* out, int channels, Int3 out_size, float scale, cudaStream_t s) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  const CrossChecks checks = read_cross_checks();
  const End end = tensor_cores() && !checks.no_fused_tail ? kFusedTail : kBlend;
  return run(Route{chunk, in_dtype, cs, end, ConvTail{nullptr, nullptr, patches, mask, out, channels, op, crop, out_size, scale}, checks},
             nb, s);
}

int Network::forward_from_host_patches(const float* h_patches, int nb, cudaStream_t s) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  CFB_CUDA(cudaMemcpyAsync(f32(kIn), h_patches, (size_t)nb * vol(patch_) * sizeof(float), cudaMemcpyHostToDevice, s));
  return run(Route{nullptr, 0, Int3{0, 0, 0}, kRawOutput, ConvTail{}, read_cross_checks()}, nb, s);
}

void Network::crop_mask(Int3 op, Int3 crop, const float* mask, int nb, float* dst, int channels, cudaStream_t s) {
  launch_crop_mask(f32(kOut), cnet_, patch_, op, crop, mask, nb, dst, channels, /*repeat=*/false, s);
}

void Network::copy_raw_output_to_host(float* h_out, cudaStream_t s) {
  CFB_CUDA(cudaMemcpyAsync(h_out, f32(kOut), (size_t)cnet_ * vol(patch_) * sizeof(float), cudaMemcpyDeviceToHost, s));
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
  if (tensor_cores()) {
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
