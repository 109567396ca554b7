// Device-side U-Net of depth 2 to 4: the generated layer table, weight packing, workspace and layer dispatch.
#include "network.cuh"

#include <cstdlib>

#include "chunkflow_b200.h"
#include "kernels_memory.cuh"
#include "kernels_simt.cuh"

namespace cfb {

int Network::taps(Op op) { return op == kOpConvT ? 4 : op == kOpHead ? 1 : 27; }

// enc0 .. enc{d-1} down, with a (1,2,2) max pool after every level but the last; up{k} + dec{k} from level d-2 up to 0,
// each decoder concatenating its transposed convolution with the encoder output of the same level; the 1x1x1 head.
std::vector<Network::Step> Network::make_steps(int depth, int& acts) {
  std::vector<Step> s;
  acts = 2;  // kIn, kOut
  auto act = [&] { return acts++; };
  std::vector<Act> enc(depth), pooled(depth, kNoAct);
  for (int k = 0; k < depth; ++k) {
    const int w = 16 << k, last = k == depth - 1;
    const Act mid = act();
    if (k == 0) s.push_back({"enc0.0", kOpFirst, 1, w, kIn, kNoAct, mid, kNoAct, 0});
    else s.push_back({"enc" + std::to_string(k) + ".0", kOpConv3, w / 2, w, pooled[k - 1], kNoAct, mid, kNoAct, k});
    enc[k] = act();
    if (!last) pooled[k] = act();
    s.push_back({"enc" + std::to_string(k) + ".2", last ? kOpConv3 : kOpConv3Pool, w, w, mid, kNoAct, enc[k], pooled[k], k});
  }
  Act below = enc[depth - 1];
  for (int k = depth - 2; k >= 0; --k) {
    const int w = 16 << k;
    const Act up = act(), mid = act(), dec = act();
    s.push_back({"up" + std::to_string(k), kOpConvT, 2 * w, w, below, kNoAct, up, kNoAct, k + 1});
    s.push_back({"dec" + std::to_string(k) + ".0", kOpConv3, 2 * w, w, up, enc[k], mid, kNoAct, k});
    s.push_back({"dec" + std::to_string(k) + ".2", kOpConv3, w, w, mid, kNoAct, dec, kNoAct, k});
    below = dec;
  }
  s.push_back({"head", kOpHead, 16, -1, below, kNoAct, kOut, kNoAct, 0});
  return s;
}

// channels of an activation: the input patches have one, every other one those of the step that produces it
int Network::act_channels(Act a) const {
  for (const Step& st : steps_)
    if (st.dst == a || st.pool == a) return st.cout;
  return 1;
}

void Network::configure(int precision, Int3 patch, int batch) {
  if (precision != CFB_PRECISION_F32_SIMT && precision != CFB_PRECISION_F16X3_UMMA && precision != CFB_PRECISION_F16_UMMA &&
      precision != CFB_PRECISION_F16F8_UMMA)
    throw std::invalid_argument("unknown precision mode");
  precision_ = precision;
  patch_ = patch;
  batch_ = batch;
}

void Network::release() {
  for (DeviceBuffer& a : act_) a.reset();
  for (ConvLayer& L : layers_) { cudaFree(L.w); cudaFree(L.bias); free_packed(L.packed); }
  layers_.clear();
  for (cudaEvent_t e : prof_pool_) cudaEventDestroy(e);
  prof_pool_.clear();
  ready_ = false;
}

float* Network::patch_input_buffer(int nb) {
  if (nb > batch_) throw std::invalid_argument("batch larger than configured");
  act_[kIn].grow((size_t)vol(patch_) * batch_ * sizeof(float));
  return f32(kIn);
}

void Network::allocate() {
  if (act_[kOut]) return;
  patch_input_buffer(1);
  auto alloc = [&](Act a, size_t bytes_per_voxel, int level) {
    act_[a].grow(bytes_per_voxel * (size_t)(vol(patch_) >> (2 * level)) * batch_);
  };
  alloc(kOut, sizeof(float) * std::max(cnet_, 1), 0);
  const size_t bytes = tensor_cores() ? sizeof(__half) * parts() : sizeof(float);  // per channel and voxel
  for (const Step& st : steps_) {
    if (st.op == kOpHead) continue;
    alloc(st.dst, bytes * st.cout, st.op == kOpConvT ? st.level - 1 : st.level);
    if (st.pool != kNoAct) alloc(st.pool, bytes * st.cout, st.level + 1);
  }
}

bool Network::load(const std::map<std::string, std::vector<float>>& host_w, int num_output_channels, std::string& err) {
  ready_ = false;
  for (ConvLayer& L : layers_) { cudaFree(L.w); cudaFree(L.bias); free_packed(L.packed); }
  layers_.clear();
  // the depth is the number of encoder levels in the state dict, and level k must be 16 << k channels wide
  int depth = 0;
  while (host_w.count("enc" + std::to_string(depth) + ".0.weight")) ++depth;
  if (depth < 2 || depth > 4) {
    err = "the U-Net depth must be 2, 3 or 4 (encoder levels enc0.0 .. enc{d-1}.0 in the state dict), found " + std::to_string(depth);
    return false;
  }
  for (int k = 0, cin = 1; k < depth; cin = 16 << k, ++k) {
    const size_t n = host_w.at("enc" + std::to_string(k) + ".0.weight").size();
    if (n != (size_t)cin * (16 << k) * 27) {
      err = "the U-Net widths must be 16, 32, 64, 128 (level k: 16 << k channels): enc" + std::to_string(k) + ".0.weight has " +
            std::to_string(n) + " values, expected " + std::to_string((size_t)cin * (16 << k) * 27);
      return false;
    }
  }
  const int align = 1 << (depth - 1);
  if (patch_.y % align || patch_.x % align) {
    err = "the " + std::to_string(depth) + "-level U-Net pools (1,2,2) " + std::to_string(depth - 1) +
          " times: patch y and x must be multiples of " + std::to_string(align);
    return false;
  }
  int acts = 0;
  std::vector<Step> steps = make_steps(depth, acts);
  if (depth != depth_) {  // a different table: new activation buffers (the staged input patches stay)
    for (size_t i = 1; i < act_.size(); ++i) act_[i].reset();
    act_.resize(acts);
  }
  depth_ = depth;
  steps_ = std::move(steps);
  for (const Step& st : steps_) {
    const std::string wn = st.name + ".weight", bn = st.name + ".bias";
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
  blend.head_w = layers_.back().w;
  blend.head_b = layers_.back().bias;
  int launches = 0;
  auto issue = [&](const char* name, auto&& launch) {
    prof_begin(name, s);
    launch();
    prof_end(s);
    ++launches;
  };
  for (size_t i = 0; i < steps_.size(); ++i) {
    const Step& st = steps_[i];
    const ConvLayer& L = layers_[i];
    const Int3 sz{patch_.z, patch_.y >> st.level, patch_.x >> st.level};
    const int cb = st.b == kNoAct ? 0 : act_channels(st.b), ca = st.cin - cb;
    if (st.op == kOpFirst) {
      if (!tc && r.chunk)
        issue("extract", [&] { launch_extract_patches(r.chunk, r.in_dtype, r.chunk_size, blend.patches, nb, patch_, f32(kIn), s); });
      issue(st.name.c_str(), [&] {
        if (!tc) launch_conv3_f32(f32(kIn), 1, nullptr, 0, L.w, L.bias, f32(st.dst), st.cout, nb, sz, /*relu=*/true, s);
        else if (r.chunk) launch_first_conv_cp8(r.chunk, r.in_dtype, r.chunk_size, blend.patches, nb, sz, first_w_, cp8(st.dst), P, s);
        else launch_first_conv_cp8_from_patches(f32(kIn), nb, sz, first_w_, cp8(st.dst), P, s);
      });
    } else if (st.op == kOpConv3 || st.op == kOpConv3Pool) {
      const bool pool = st.op == kOpConv3Pool, fuse_pool = tc && pool && !r.checks.no_pool_fusion;
      const bool fuse_tail = r.end == kFusedTail && steps_[i + 1].op == kOpHead;  // + head + sigmoid + crop + mask + blend
      issue(fuse_tail ? (st.name + "+head+blend").c_str() : st.name.c_str(), [&] {
        if (!tc) launch_conv3_f32(f32(st.a), ca, cb ? f32(st.b) : nullptr, cb, L.w, L.bias, f32(st.dst), st.cout, nb, sz, true, s);
        else launch_conv3_wgmma(cp8(st.a), ca, cb ? cp8(st.b) : nullptr, cb, L.packed, cp8(st.dst), nb, sz, /*relu=*/true, s,
                                fuse_tail ? &blend : nullptr, fuse_pool ? cp8(st.pool) : nullptr);
      });
      if (tc && st.cout > 64) ++launches;  // a 128-channel layer: one launch per 64-channel half (kernels_wgmma_wide.cu)
      if (pool && !fuse_pool)
        issue(("pool" + std::to_string(st.level)).c_str(), [&] {
          if (tc) launch_maxpool_cp8(cp8(st.dst), cp8(st.pool), st.cout, P, nb, sz, s);
          else launch_maxpool_f32(f32(st.dst), f32(st.pool), st.cout, nb, sz, s);
        });
    } else if (st.op == kOpConvT) {
      issue(st.name.c_str(), [&] {
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
      issue(st.name.c_str(), [&] {
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
  const int64_t v = vol(size);
  DeviceBuffer in((size_t)cin * v * 4), w((size_t)cout * cin * 27 * 4), b((size_t)cout * 4), out((size_t)cout * v * 4);
  float *d_in = in.as<float>(), *d_out = out.as<float>();
  CFB_CUDA(cudaMemcpyAsync(d_in, h_in, (size_t)cin * v * 4, cudaMemcpyHostToDevice, s));
  CFB_CUDA(cudaMemcpyAsync(w.as(), h_w, (size_t)cout * cin * 27 * 4, cudaMemcpyHostToDevice, s));
  CFB_CUDA(cudaMemcpyAsync(b.as(), h_b, (size_t)cout * 4, cudaMemcpyHostToDevice, s));
  if (tensor_cores()) {
    if (cin % 16) throw std::runtime_error("the wgmma convolution needs cin % 16 == 0");
    const int P = parts();
    DeviceBuffer cp8_in((size_t)cin * P * v * 2), cp8_out((size_t)cout * P * v * 2);
    __half *c_in = cp8_in.as<__half>(), *c_out = cp8_out.as<__half>();
    PackedConv pk;
    pack_conv3_weights(h_w, h_b, cin, cout, fmt(), pk);
    launch_planar_to_cp8(d_in, c_in, cin, fmt(), 1, size, s);
    // exercise the two-source (concat) path whenever the channel count allows it
    const int ca = cin >= 32 ? cin / 2 : cin, cb = cin - ca;
    launch_conv3_wgmma(c_in, ca, cb ? c_in + (size_t)ca * P * v : nullptr, cb, pk, c_out, 1, size, relu, s);
    launch_cp8_to_planar(c_out, d_out, cout, fmt(), 1, size, s);
    CFB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)cout * v * 4, cudaMemcpyDeviceToHost, s));
    cudaError_t err = cudaStreamSynchronize(s);
    free_packed(pk);
    CFB_CUDA(err);
    return CFB_OK;
  }
  launch_conv3_f32(d_in, cin, nullptr, 0, w.as<float>(), b.as<float>(), d_out, cout, 1, size, relu, s);
  CFB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)cout * v * 4, cudaMemcpyDeviceToHost, s));
  CFB_CUDA(cudaStreamSynchronize(s));
  return CFB_OK;
}

}  // namespace cfb
