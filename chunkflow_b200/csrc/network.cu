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

int Network::debug_layer(const cfb_layer_args& a, cudaStream_t s) {
  const int nb = a.nb, ca = a.ca, cb = a.cb, cin = a.ca + a.cb, cout = a.cout, hc = a.head_channels;
  const Int3 sz{a.size[0], a.size[1], a.size[2]}, half_sz{sz.z, sz.y / 2, sz.x / 2}, double_sz{sz.z, 2 * sz.y, 2 * sz.x};
  const Int3 op{a.out_patch[0], a.out_patch[1], a.out_patch[2]}, crop{a.crop[0], a.crop[1], a.crop[2]};
  const Int3 os{a.out_size[0], a.out_size[1], a.out_size[2]}, cs{a.chunk_size[0], a.chunk_size[1], a.chunk_size[2]};
  if (nb < 1 || sz.z < 1 || sz.y < 1 || sz.x < 1 || ca < 0 || cb < 0) throw std::invalid_argument("debug_layer: bad shape");
  const bool tc = tensor_cores(), first_from_chunk = a.op == CFB_LAYER_FIRST && a.chunk;
  const bool blend = a.op == CFB_LAYER_HEAD_BLEND || a.op == CFB_LAYER_CONV3_HEAD_BLEND;
  const bool head = blend || a.op == CFB_LAYER_HEAD_SIGMOID;
  if ((a.op == CFB_LAYER_CONV3_POOL || a.op == CFB_LAYER_MAXPOOL) && ((sz.y & 1) || (sz.x & 1)))
    throw std::invalid_argument("debug_layer: pooling needs even y and x");
  if (a.op == CFB_LAYER_FIRST && (ca != 1 || cb)) throw std::invalid_argument("debug_layer: the first layer reads one channel");
  if (head && (hc < 1 || hc > 8)) throw std::invalid_argument("debug_layer: 1 to 8 head channels");
  if (blend && (!a.mask || !a.out_origins || vol(op) < 1 || vol(os) < 1 || op.z + crop.z > sz.z || op.y + crop.y > sz.y ||
                op.x + crop.x > sz.x || crop.z < 0 || crop.y < 0 || crop.x < 0))
    throw std::invalid_argument("debug_layer: bad blend geometry");
  const CrossChecks checks = read_cross_checks();
  const int F = fmt(), P = parts();

  std::vector<DeviceBuffer> bufs;  // every allocation of this call
  auto alloc = [&](size_t bytes) { bufs.emplace_back(bytes); return bufs.back().as(); };
  auto upload = [&](const void* h, size_t bytes) {
    if (!h) throw std::invalid_argument("debug_layer: missing input array");
    void* d = alloc(bytes);
    CFB_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
    return static_cast<float*>(d);
  };
  auto download = [&](float* h, const float* d, size_t bytes) {
    if (!h) throw std::invalid_argument("debug_layer: missing output array");
    CFB_CUDA(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s));
  };
  // planar fp32 (nb, c, e) <-> CP8 of the mode's format; 128 channels half-major (kernels_conv.cuh): one conversion per
  // (half, patch)
  auto to_cp8 = [&](const float* d, int c, Int3 e) {
    if (c % 8 || (c > 64 && c != 128)) throw std::invalid_argument("debug_layer: CP8 tensors have 8 .. 64 or 128 channels");
    __half* t = static_cast<__half*>(alloc((size_t)nb * c * P * vol(e) * sizeof(__half)));
    if (c <= 64) launch_planar_to_cp8(d, t, c, F, nb, e, s);
    else
      for (int h = 0; h < 2; ++h)
        for (int b = 0; b < nb; ++b)
          launch_planar_to_cp8(d + ((size_t)b * c + h * 64) * vol(e), t + ((size_t)h * nb + b) * 64 * P * vol(e), 64, F, 1, e, s);
    return t;
  };
  auto from_cp8 = [&](const __half* t, int c, Int3 e) {
    float* d = static_cast<float*>(alloc((size_t)nb * c * vol(e) * sizeof(float)));
    if (c <= 64) launch_cp8_to_planar(t, d, c, F, nb, e, s);
    else
      for (int h = 0; h < 2; ++h)
        for (int b = 0; b < nb; ++b)
          launch_cp8_to_planar(t + ((size_t)h * nb + b) * 64 * P * vol(e), d + ((size_t)b * c + h * 64) * vol(e), 64, F, 1, e, s);
    return d;
  };
  auto cp8_out = [&](int c, Int3 e) { return static_cast<__half*>(alloc((size_t)nb * c * P * vol(e) * sizeof(__half))); };
  auto f32_out = [&](int c, Int3 e) { return static_cast<float*>(alloc((size_t)nb * c * vol(e) * sizeof(float))); };
  struct Packed {
    PackedConv p;
    ~Packed() { free_packed(p); }
  } pk;

  const float* d_a = first_from_chunk ? nullptr : upload(a.a, (size_t)nb * ca * vol(sz) * sizeof(float));
  const float* d_b = cb ? upload(a.b, (size_t)nb * cb * vol(sz) * sizeof(float)) : nullptr;
  const __half* c_a = tc && a.op != CFB_LAYER_FIRST ? to_cp8(d_a, ca, sz) : nullptr;
  const __half* c_b = tc && cb ? to_cp8(d_b, cb, sz) : nullptr;
  const float* d_hw = head ? upload(a.head_weight, (size_t)hc * 16 * sizeof(float)) : nullptr;
  const float* d_hb = head ? upload(a.head_bias, (size_t)hc * sizeof(float)) : nullptr;
  PatchPos* d_pp = nullptr;
  if (blend || first_from_chunk) {
    std::vector<PatchPos> pp(nb);
    for (int b = 0; b < nb; ++b) {
      if (first_from_chunk) {
        pp[b].iz = a.in_origins[3 * b]; pp[b].iy = a.in_origins[3 * b + 1]; pp[b].ix = a.in_origins[3 * b + 2];
        if (pp[b].iz < 0 || pp[b].iy < 0 || pp[b].ix < 0 || pp[b].iz + sz.z > cs.z || pp[b].iy + sz.y > cs.y || pp[b].ix + sz.x > cs.x)
          throw std::invalid_argument("debug_layer: patch outside the chunk");
      }
      if (blend) { pp[b].oz = a.out_origins[3 * b]; pp[b].oy = a.out_origins[3 * b + 1]; pp[b].ox = a.out_origins[3 * b + 2]; }
    }
    d_pp = reinterpret_cast<PatchPos*>(upload(pp.data(), nb * sizeof(PatchPos)));
  }
  float* d_out = nullptr;   // blend: the accumulated output chunk
  const float* d_mask = nullptr;
  if (blend) {
    d_mask = upload(a.mask, vol(op) * sizeof(float));
    d_out = upload(a.out, (size_t)hc * vol(os) * sizeof(float));
  }
  auto blend_tail = [&]() { return ConvTail{d_hw, d_hb, d_pp, d_mask, d_out, hc, op, crop, os, a.scale}; };

  switch (a.op) {
    case CFB_LAYER_CONV3: case CFB_LAYER_CONV3_POOL: case CFB_LAYER_CONV3_HEAD_BLEND: {
      const bool pool = a.op == CFB_LAYER_CONV3_POOL, tail = a.op == CFB_LAYER_CONV3_HEAD_BLEND;
      if (tail && (cin != 16 || cout != 16)) throw std::invalid_argument("debug_layer: the fused tail follows a 16 -> 16 layer");
      const bool relu = tail || a.relu;
      if (!tc) {
        const float *w = upload(a.weight, (size_t)cout * cin * 27 * sizeof(float)), *bias = upload(a.bias, cout * sizeof(float));
        float* o = f32_out(cout, sz);
        launch_conv3_f32(d_a, ca, d_b, cb, w, bias, o, cout, nb, sz, relu, s);
        if (tail) {
          float* net = f32_out(hc, sz);
          launch_head_sigmoid_f32(o, d_hw, d_hb, net, 16, hc, nb, sz, s);
          launch_blend_patches(net, hc, sz, op, crop, d_mask, d_pp, nb, d_out, hc, os, a.scale, s);
          break;
        }
        download(a.out, o, (size_t)nb * cout * vol(sz) * sizeof(float));
        if (pool) {
          float* po = f32_out(cout, half_sz);
          launch_maxpool_f32(o, po, cout, nb, sz, s);
          download(a.pooled, po, (size_t)nb * cout * vol(half_sz) * sizeof(float));
        }
        break;
      }
      if (!a.weight || !a.bias) throw std::invalid_argument("debug_layer: missing weights");
      pack_conv3_weights(a.weight, a.bias, cin, cout, F, pk.p);
      __half* o = cp8_out(cout, sz);
      __half* po = pool ? cp8_out(cout, half_sz) : nullptr;
      const ConvTail t = blend_tail();
      const bool fuse_tail = tail && !checks.no_fused_tail, fuse_pool = pool && !checks.no_pool_fusion;
      launch_conv3_wgmma(c_a, ca, c_b, cb, pk.p, o, nb, sz, relu, s, fuse_tail ? &t : nullptr, fuse_pool ? po : nullptr);
      if (tail) {
        if (!fuse_tail) launch_head_blend_cp8(o, d_hw, d_hb, 16, hc, F, sz, op, crop, d_mask, d_pp, nb, d_out, hc, os, a.scale, s);
        break;
      }
      download(a.out, from_cp8(o, cout, sz), (size_t)nb * cout * vol(sz) * sizeof(float));
      if (pool) {
        if (!fuse_pool) launch_maxpool_cp8(o, po, cout, F, nb, sz, s);
        download(a.pooled, from_cp8(po, cout, half_sz), (size_t)nb * cout * vol(half_sz) * sizeof(float));
      }
      break;
    }
    case CFB_LAYER_CONVT: {
      const float *w = upload(a.weight, (size_t)ca * cout * 4 * sizeof(float)), *bias = upload(a.bias, cout * sizeof(float));
      if (!tc) {
        float* o = f32_out(cout, double_sz);
        launch_convT_f32(d_a, w, bias, o, ca, cout, nb, sz, s);
        download(a.out, o, (size_t)nb * cout * vol(double_sz) * sizeof(float));
        break;
      }
      __half* o = cp8_out(cout, double_sz);
      if (checks.simt_convt) {
        launch_convT_cp8(c_a, w, bias, o, ca, cout, F, nb, sz, s);
      } else {
        pack_convT_weights(a.weight, a.bias, ca, cout, F, pk.p);
        launch_convT_wgmma(c_a, pk.p, o, nb, sz, s);
      }
      download(a.out, from_cp8(o, cout, double_sz), (size_t)nb * cout * vol(double_sz) * sizeof(float));
      break;
    }
    case CFB_LAYER_MAXPOOL: {
      if (!tc) {
        float* o = f32_out(ca, half_sz);
        launch_maxpool_f32(d_a, o, ca, nb, sz, s);
        download(a.out, o, (size_t)nb * ca * vol(half_sz) * sizeof(float));
        break;
      }
      __half* o = cp8_out(ca, half_sz);
      launch_maxpool_cp8(c_a, o, ca, F, nb, sz, s);
      download(a.out, from_cp8(o, ca, half_sz), (size_t)nb * ca * vol(half_sz) * sizeof(float));
      break;
    }
    case CFB_LAYER_FIRST: {
      if (!a.weight || !a.bias) throw std::invalid_argument("debug_layer: missing weights");
      const void* chunk = nullptr;
      if (first_from_chunk) {
        if (a.chunk_dtype != CFB_DTYPE_U8 && a.chunk_dtype != CFB_DTYPE_F32) throw std::invalid_argument("debug_layer: uint8 or float32 chunk");
        chunk = upload(a.chunk, vol(cs) * (a.chunk_dtype == CFB_DTYPE_U8 ? 1 : sizeof(float)));
      }
      if (!tc) {
        const float *w = upload(a.weight, 16 * 27 * sizeof(float)), *bias = upload(a.bias, 16 * sizeof(float));
        const float* in = d_a;
        if (chunk) {
          if (sz.x % 4) throw std::invalid_argument("debug_layer: the patch extraction needs x % 4 == 0");
          float* ex = f32_out(1, sz);
          launch_extract_patches(chunk, a.chunk_dtype, cs, d_pp, nb, sz, ex, s);
          in = ex;
        }
        float* o = f32_out(16, sz);
        launch_conv3_f32(in, 1, nullptr, 0, w, bias, o, 16, nb, sz, /*relu=*/true, s);
        download(a.out, o, (size_t)nb * 16 * vol(sz) * sizeof(float));
        break;
      }
      FirstConvW W{};
      for (int t = 0; t < 27; ++t)
        for (int c = 0; c < 16; ++c) W.w[t][c] = a.weight[c * 27 + t];
      for (int c = 0; c < 16; ++c) W.b[c] = a.bias[c];
      __half* o = cp8_out(16, sz);
      if (chunk) launch_first_conv_cp8(chunk, a.chunk_dtype, cs, d_pp, nb, sz, W, o, F, s);
      else launch_first_conv_cp8_from_patches(d_a, nb, sz, W, o, F, s);
      download(a.out, from_cp8(o, 16, sz), (size_t)nb * 16 * vol(sz) * sizeof(float));
      break;
    }
    case CFB_LAYER_HEAD_SIGMOID: case CFB_LAYER_HEAD_BLEND: {
      if (ca != 16 || cb) throw std::invalid_argument("debug_layer: the head reads 16 channels");
      float* net = f32_out(hc, sz);
      if (a.op == CFB_LAYER_HEAD_BLEND && tc) {
        launch_head_blend_cp8(c_a, d_hw, d_hb, 16, hc, F, sz, op, crop, d_mask, d_pp, nb, d_out, hc, os, a.scale, s);
        break;
      }
      if (tc) launch_head_sigmoid_cp8(c_a, d_hw, d_hb, net, 16, hc, F, nb, sz, s);
      else launch_head_sigmoid_f32(d_a, d_hw, d_hb, net, 16, hc, nb, sz, s);
      if (a.op == CFB_LAYER_HEAD_BLEND) launch_blend_patches(net, hc, sz, op, crop, d_mask, d_pp, nb, d_out, hc, os, a.scale, s);
      else download(a.out, net, (size_t)nb * hc * vol(sz) * sizeof(float));
      break;
    }
    case CFB_LAYER_ROUND_TRIP:
      if (!tc) throw std::invalid_argument("debug_layer: the simt mode keeps fp32 activations");
      download(a.out, from_cp8(c_a, ca, sz), (size_t)nb * ca * vol(sz) * sizeof(float));
      break;
    default:
      throw std::invalid_argument("debug_layer: unknown op");
  }
  if (blend) download(a.out, d_out, (size_t)hc * vol(os) * sizeof(float));
  CFB_CUDA(cudaStreamSynchronize(s));
  return CFB_OK;
}

}  // namespace cfb
