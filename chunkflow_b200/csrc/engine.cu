// chunkflow_b200 engine: C-ABI entry points (include/chunkflow_b200.h) and the per-chunk
// orchestration of the inference hot path.  Host logic restates the reference's geometry
// (chunkflow/flow/divid_conquer/inferencer.py) -- all arithmetic on voxels runs in CUDA
// kernels; there is no CPU fallback.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"
#include "host_stager.cuh"
#include "kernels_memory.cuh"
#include "kernels_simt.cuh"
#include "network.cuh"

namespace cfb {

static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }

// ---- patch mask (reference patch/patch_mask.py:15-68), fp64 on the host, once ------------
static std::vector<float> build_patch_mask(Int3 p, Int3 ov) {
  const int64_t n = vol(p);
  std::vector<double> bump(n);
  auto coord = [](int i, int len) { return (i + 1.0) / (len + 1.0) * 2.0 - 1.0; };
  std::vector<double> tz(p.z), ty(p.y), tx(p.x);
  for (int i = 0; i < p.z; ++i) { double c = coord(i, p.z); tz[i] = -1.0 / (1.0 - c * c); }
  for (int i = 0; i < p.y; ++i) { double c = coord(i, p.y); ty[i] = -1.0 / (1.0 - c * c); }
  for (int i = 0; i < p.x; ++i) { double c = coord(i, p.x); tx[i] = -1.0 / (1.0 - c * c); }
  double bmin = INFINITY, bmax = -INFINITY;
  for (int z = 0; z < p.z; ++z)
    for (int y = 0; y < p.y; ++y)
      for (int x = 0; x < p.x; ++x) {
        // same association as numpy: (fx + fy) + fz
        double v = std::exp((tx[x] + ty[y]) + tz[z]);
        bump[((int64_t)z * p.y + y) * p.x + x] = v;
        bmin = std::min(bmin, v);
        bmax = std::max(bmax, v);
      }
  // np.interp(b, (min, max), (1, 1e6))
  const double slope = (1e6 - 1.0) / (bmax - bmin);
  for (auto& v : bump) v = (v >= bmax) ? 1e6 : slope * (v - bmin) + 1.0;
  // 3x3x3 neighbour simulation at the nominal stride; accumulation order nz, ny, nx ascending
  const Int3 st{p.z - ov.z, p.y - ov.y, p.x - ov.x};
  std::vector<float> mask(n);
  for (int z = 0; z < p.z; ++z)
    for (int y = 0; y < p.y; ++y)
      for (int x = 0; x < p.x; ++x) {
        double sum = 0.0;
        for (int nz = 0; nz < 3; ++nz) {
          int lz = z + st.z - nz * st.z;  // coordinate inside neighbour nz
          if (lz < 0 || lz >= p.z) continue;
          for (int ny = 0; ny < 3; ++ny) {
            int ly = y + st.y - ny * st.y;
            if (ly < 0 || ly >= p.y) continue;
            for (int nx = 0; nx < 3; ++nx) {
              int lx = x + st.x - nx * st.x;
              if (lx < 0 || lx >= p.x) continue;
              sum += bump[((int64_t)lz * p.y + ly) * p.x + lx];
            }
          }
        }
        const int64_t i = ((int64_t)z * p.y + y) * p.x + x;
        mask[i] = (float)(bump[i] / sum);
      }
  return mask;
}

struct AxisGrid {
  std::vector<int> in_start;   // chunk-local input starts
  std::vector<int> out_start;  // output-buffer coordinates of the cropped output patch
};

// reference inferencer.py:268-283: range(0, size - overlap, stride), last start clamped back
static AxisGrid axis_grid(int size, int ip, int ioverlap, int istride, int pcrop, int out_offset) {
  AxisGrid g;
  for (int i = 0; i < size - ioverlap; i += istride) {
    int s = i;
    if (s + ip > size) s = size - ip;
    g.in_start.push_back(s);
    g.out_start.push_back(s + pcrop - out_offset);
  }
  return g;
}

// The patch grid on one chunk shape (reference inferencer.py:183-204,255-292).
struct ChunkGeometry {
  Int3 size{0, 0, 0};  // the input chunk
  Int3 out{0, 0, 0};   // the output buffer: the chunk less the output crop margin on either side
  AxisGrid z, y, x;
};

}  // namespace cfb

using namespace cfb;

struct cfb_engine {
  cfb_params p{};
  std::string device_name;
  Int3 ip{}, op{}, ovl{}, ocm{}, pcrop{}, istride{}, ioverlap{};
  std::map<std::string, std::vector<float>> host_w;
  Network net;
  std::vector<float> h_mask;
  DeviceBuffer mask;

  // per-chunk-shape cache (prepare_chunk; the reference caches its output_chunk_mask the same way, :300-312)
  ChunkGeometry geo;
  std::vector<PatchPos> h_patches;
  DeviceBuffer patches;
  DeviceBuffer cover_tables;  // `cover` points into it
  CoverTables cover{};
  DeviceBuffer winv;          // 1/W of `geo`, computed on first use (inverse_weight)
  DeviceBuffer slab_cover_tables;

  DeviceBuffer flags;  // unsigned int [0] nonzero flag, [1] max bits
  cudaStream_t own_stream = nullptr;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_ready = nullptr;
  DeviceBuffer host_in, host_out, plugin_out, plugin_in;
  bool plugin_active = false; int plugin_dtype = 0;

  std::unique_ptr<HostStager> stager;  // pinned ring + host threads for results that go to pageable memory

  cudaEvent_t ev[8]{};
  bool timing_valid = false;
  int64_t launches = 0;

  // reference transform.py:114-156: 8 augmented evaluations per patch, averaged.  CFB_AUGMENT_REFERENCE: the
  // reference's flips act on the channel / batch axes, so its 8 variants are 2 network evaluations (identity,
  // transpose), each blended with its channel-reversed copy (weight 1/4); CFB_AUGMENT_SPATIAL: 8 spatial variants.
  int variants() const {
    if (!p.augment || p.framework != CFB_FRAMEWORK_UNET3L) return 1;
    return p.augment == CFB_AUGMENT_SPATIAL ? 8 : 2;
  }
  int variant_flags(int v) const { return (p.augment == CFB_AUGMENT_REFERENCE && variants() > 1) ? (v | kTtaChannelSym) : v; }
  float variant_scale() const { return variants() == 1 ? 1.0f : (p.augment == CFB_AUGMENT_SPATIAL ? 0.125f : 0.25f); }

  // Every entry point that takes a chunk shape checks it here, in this order.
  ChunkGeometry geometry(int64_t cz, int64_t cy, int64_t cx) const {
    if (cz < ip.z || cy < ip.y || cx < ip.x) throw std::invalid_argument("input chunk is smaller than the input patch");
    if (cz > INT32_MAX || cy > INT32_MAX || cx > INT32_MAX) throw std::invalid_argument("chunk too large");
    ChunkGeometry g;
    g.size = Int3{(int)cz, (int)cy, (int)cx};
    g.out = Int3{g.size.z - 2 * ocm.z, g.size.y - 2 * ocm.y, g.size.x - 2 * ocm.x};  // inferencer.py:194-196
    if (g.out.z <= 0 || g.out.y <= 0 || g.out.x <= 0) throw std::invalid_argument("output crop margin swallows the chunk");
    g.z = axis_grid(g.size.z, ip.z, ioverlap.z, istride.z, pcrop.z, ocm.z);
    g.y = axis_grid(g.size.y, ip.y, ioverlap.y, istride.y, pcrop.y, ocm.y);
    g.x = axis_grid(g.size.x, ip.x, ioverlap.x, istride.x, pcrop.x, ocm.x);
    return g;
  }

  ~cfb_engine() {
    cudaSetDevice(p.device);  // the DeviceBuffer members are freed after this body, on this device
    stager.reset();
    net.release();
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (own_stream) cudaStreamDestroy(own_stream);
    if (copy_stream) cudaStreamDestroy(copy_stream);
    if (ev_ready) cudaEventDestroy(ev_ready);
  }
};

namespace {

// Appends the cover table of one output axis, counting the patch axis-indices [row_begin, row_end): for every
// coordinate the covering indices ascending, then -1 up to kMaxCover entries.
void append_cover(const AxisGrid& g, int op_len, int out_len, int row_begin, int row_end, std::vector<int>& t) {
  const size_t base = t.size();
  t.resize(base + (size_t)out_len * kMaxCover, -1);
  for (int v = 0; v < out_len; ++v) {
    int n = 0;
    for (int k = row_begin; k < row_end; ++k) {
      if (g.out_start[k] <= v && v < g.out_start[k] + op_len) {
        if (n == kMaxCover) throw std::runtime_error("a voxel is covered by more than 4 patches along one axis (overlap too large)");
        t[base + (size_t)v * kMaxCover + n++] = k;
      }
    }
  }
}

// Builds the weight-volume tables of `g` in one host array, in the order of CoverTables, and uploads it into `buf`.
// The z cover table counts the patch z-rows [row_begin, row_end) only: those of one slab.
CoverTables upload_cover_tables(const ChunkGeometry& g, Int3 op, DeviceBuffer& buf, cudaStream_t s, int row_begin = 0,
                                int row_end = -1) {
  if (row_end < 0) row_end = (int)g.z.out_start.size();
  std::vector<int> host;
  append_cover(g.z, op.z, g.out.z, row_begin, row_end, host);
  append_cover(g.y, op.y, g.out.y, 0, (int)g.y.out_start.size(), host);
  append_cover(g.x, op.x, g.out.x, 0, (int)g.x.out_start.size(), host);
  for (const AxisGrid* a : {&g.z, &g.y, &g.x}) host.insert(host.end(), a->out_start.begin(), a->out_start.end());
  buf.grow(host.size() * sizeof(int));
  CFB_CUDA(cudaMemcpyAsync(buf.as(), host.data(), host.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CFB_CUDA(cudaStreamSynchronize(s));  // `host` is a temporary
  CoverTables t;
  t.cover_z = buf.as<int>();
  t.cover_y = t.cover_z + (size_t)g.out.z * kMaxCover;
  t.cover_x = t.cover_y + (size_t)g.out.y * kMaxCover;
  t.ostart_z = t.cover_x + (size_t)g.out.x * kMaxCover;
  t.ostart_y = t.ostart_z + g.z.out_start.size();
  t.ostart_x = t.ostart_y + g.y.out_start.size();
  return t;
}

void prepare_chunk(cfb_engine* e, int64_t cz, int64_t cy, int64_t cx, cudaStream_t s) {
  ChunkGeometry g = e->geometry(cz, cy, cx);  // checked before the cache: an empty cache holds the shape (0, 0, 0)
  if (e->geo.size.z == g.size.z && e->geo.size.y == g.size.y && e->geo.size.x == g.size.x) return;
  e->geo = ChunkGeometry{};  // no shape is cached until its tables are on the device
  // Freed, not reused in place: cudaFree waits for the kernels of earlier calls, on any stream, that may still read them.
  e->winv.reset();
  e->patches.reset();
  e->cover_tables.reset();
  e->h_patches.clear();
  for (size_t a = 0; a < g.z.in_start.size(); ++a)
    for (size_t b = 0; b < g.y.in_start.size(); ++b)
      for (size_t c = 0; c < g.x.in_start.size(); ++c)
        for (int v = 0; v < e->variants(); ++v)  // 8 flip/transpose variants per patch with --augment
          e->h_patches.push_back(PatchPos{g.z.in_start[a], g.y.in_start[b], g.x.in_start[c],
                                          g.z.out_start[a], g.y.out_start[b], g.x.out_start[c], e->variant_flags(v)});
  const size_t bytes = e->h_patches.size() * sizeof(PatchPos);
  e->patches.grow(bytes);
  CFB_CUDA(cudaMemcpyAsync(e->patches.as(), e->h_patches.data(), bytes, cudaMemcpyHostToDevice, s));
  e->cover = upload_cover_tables(g, e->op, e->cover_tables, s);
  e->geo = std::move(g);
}

const float* inverse_weight(cfb_engine* e, cudaStream_t s) {
  if (!e->winv) {
    DeviceBuffer w(vol(e->geo.out) * sizeof(float));
    launch_weight_volume(e->mask.as<float>(), e->op, e->cover, e->geo.out, w.as<float>(), /*invert=*/true, s);
    e->launches++;
    e->winv = std::move(w);
  }
  return e->winv.as<float>();
}

// a6 on an empty accumulator: clears the flags, tests the input chunk for a non-zero voxel and zeroes `out`, the output
// buffer of `geo`.  Returns the launches.
int start_chunk(cfb_engine* e, const void* d_in, int in_dtype, float* out, cudaStream_t s) {
  unsigned int* flags = e->flags.as<unsigned int>();
  CFB_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(unsigned int), s));
  launch_any_nonzero(d_in, in_dtype, vol(e->geo.size), flags, s);
  CFB_CUDA(cudaMemsetAsync(out, 0, (size_t)e->p.num_output_channels * vol(e->geo.out) * sizeof(float), s));
  return 1;
}

// a12 + a14 on a (channels, nvox) volume: out *= w (1/W, or W if !w_is_inverse; none without a weight) over `count` voxels
// per channel from voxel `first` (count < 0: all), tracking the maximum into the flags; then the myelin mask when it is
// configured, which needs the whole volume (the progressive download is off with it).  Returns the launches.
int finish_output(cfb_engine* e, float* out, const float* w, bool w_is_inverse, int channels, int64_t nvox, cudaStream_t s,
                  int64_t first = 0, int64_t count = -1) {
  if (e->p.has_myelin_threshold && count >= 0) throw std::logic_error("the myelin mask needs the whole output volume");
  unsigned int* flags = e->flags.as<unsigned int>();
  launch_normalize(out + first, w ? w + first : nullptr, w_is_inverse, channels, count < 0 ? nvox : count, flags + 1, flags, s,
                   nvox);
  if (!e->p.has_myelin_threshold) return 1;
  launch_myelin_mask(out, channels, nvox, e->p.mask_myelin_threshold, s);
  return 2;
}

// a13 (reference inferencer.py:465-466) when check_output_range is set: reads the maximum the normalisation tracked, which
// synchronises `s`.
int output_range_status(cfb_engine* e, cudaStream_t s) {
  if (!e->p.check_output_range) return CFB_OK;
  unsigned int flags[2];
  CFB_CUDA(cudaMemcpyAsync(flags, e->flags.as(), sizeof(flags), cudaMemcpyDeviceToHost, s));
  CFB_CUDA(cudaStreamSynchronize(s));
  float vmax;
  std::memcpy(&vmax, &flags[1], 4);
  if (vmax < 1.0001f) return CFB_OK;
  set_last_error("output buffer should not be greater than 1 (max = " + std::to_string(vmax) + ")");
  return CFB_ERR_OUTPUT_RANGE;
}

// Progressive download (host variant): output planes are final as soon as every patch z-row that
// touches them has been blended (rows are processed in ascending z), so they are normalised and
// copied to the host on a second stream while later rows are still being computed.
struct Progressive {
  float* h_out = nullptr;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ready = nullptr;
  const float* winv = nullptr;
  int planes_done = 0;
  HostStager* stager = nullptr;  // set when h_out is pageable memory
};

bool is_pinned_host(const void* p) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

void flush_planes(cfb_engine* e, Progressive* pg, float* d_out, int z_end, cudaStream_t s) {
  if (z_end <= pg->planes_done) return;
  const int C = e->p.num_output_channels;
  const int64_t plane = (int64_t)e->geo.out.y * e->geo.out.x, nvox = vol(e->geo.out);
  const int64_t off = (int64_t)pg->planes_done * plane, count = (int64_t)(z_end - pg->planes_done) * plane;
  e->launches += finish_output(e, d_out, pg->winv, true, C, nvox, s, off, count);
  if (pg->stager) {
    for (int c = 0; c < C; ++c)
      pg->stager->push(d_out + c * nvox + off, pg->h_out + c * nvox + off, (size_t)count * sizeof(float), s, pg->copy_stream);
  } else {
    CFB_CUDA(cudaEventRecord(pg->ready, s));
    CFB_CUDA(cudaStreamWaitEvent(pg->copy_stream, pg->ready, 0));
    for (int c = 0; c < C; ++c)
      CFB_CUDA(cudaMemcpyAsync(pg->h_out + c * nvox + off, d_out + c * nvox + off, (size_t)count * sizeof(float),
                               cudaMemcpyDeviceToHost, pg->copy_stream));
  }
  pg->planes_done = z_end;
}

// Runs the patch loop for patches [first, last) and accumulates into d_out.
void run_patches(cfb_engine* e, const void* d_in, int in_dtype, int64_t first, int64_t last, float* d_out,
                 cudaStream_t s, Progressive* pg = nullptr) {
  const ChunkGeometry& g = e->geo;
  const int C = e->p.num_output_channels;
  const int B = std::max(1, e->p.batch_size);
  const int64_t per_row = (int64_t)g.y.in_start.size() * g.x.in_start.size() * e->variants();
  const float scale = e->variant_scale();
  for (int64_t i = first; i < last; i += B) {
    const int nb = (int)std::min<int64_t>(B, last - i);
    if (pg) {
      // every patch of z-rows < row is launched: planes below the output start of `row` are final
      const int64_t row = i / per_row;
      if (row < (int64_t)g.z.out_start.size()) flush_planes(e, pg, d_out, std::max(0, std::min(g.z.out_start[row], g.out.z)), s);
    }
    const PatchPos* pp = e->patches.as<PatchPos>() + i;
    if (e->p.framework == CFB_FRAMEWORK_IDENTITY) {
      launch_identity_blend(d_in, in_dtype, g.size, e->ip, e->op, e->pcrop, e->mask.as<float>(), pp, nb, d_out, C, g.out, s);
      e->launches++;
    } else {
      e->launches += e->net.forward_and_blend(d_in, in_dtype, g.size, pp, nb, e->op, e->pcrop, e->mask.as<float>(), d_out, C, g.out,
                                              scale, s);
    }
  }
}

int infer_impl(cfb_engine* e, const void* d_in, int in_dtype, int64_t cz, int64_t cy, int64_t cx,
               int64_t zrow_begin, int64_t zrow_end, bool slab, float* d_out, float* d_weight, cudaStream_t s,
               Progressive* pg = nullptr) {
  if (in_dtype != CFB_DTYPE_U8 && in_dtype != CFB_DTYPE_F32) throw std::invalid_argument("unsupported input dtype");
  if (e->p.framework == CFB_FRAMEWORK_UNET3L && !e->net.ready()) {
    set_last_error("weights not committed: call cfb_set_weight for every tensor, then cfb_commit_weights");
    return CFB_ERR_WEIGHTS;
  }
  CFB_CUDA(cudaSetDevice(e->p.device));
  e->launches = 0;
  CFB_CUDA(cudaEventRecord(e->ev[0], s));
  prepare_chunk(e, cz, cy, cx, s);
  e->launches += start_chunk(e, d_in, in_dtype, d_out, s);
  const int64_t ny = e->geo.y.in_start.size(), nx = e->geo.x.in_start.size(), nz = e->geo.z.in_start.size();
  if (slab) {
    if (zrow_begin < 0 || zrow_end > nz || zrow_begin > zrow_end) throw std::invalid_argument("bad z-row range");
  } else {
    zrow_begin = 0; zrow_end = nz;
  }
  if (pg) {
    if (slab || e->p.has_myelin_threshold) pg = nullptr;  // those need the whole volume before the final pass
    else if (e->p.mask_output_chunk) pg->winv = inverse_weight(e, s);
  }
  CFB_CUDA(cudaEventRecord(e->ev[1], s));
  run_patches(e, d_in, in_dtype, zrow_begin * ny * nx * e->variants(), zrow_end * ny * nx * e->variants(), d_out, s, pg);
  CFB_CUDA(cudaEventRecord(e->ev[2], s));
  if (slab && d_weight) {
    // partial weight sum of this slab's patches only
    const CoverTables t = upload_cover_tables(e->geo, e->op, e->slab_cover_tables, s, (int)zrow_begin, (int)zrow_end);
    launch_weight_volume(e->mask.as<float>(), e->op, t, e->geo.out, d_weight, /*invert=*/false, s);
    e->launches++;
  } else if (slab) {
    // no partial weight volume wanted: the owner of a plane computes the full weight sum itself (cfb_weight_volume_device)
  } else if (pg) {
    flush_planes(e, pg, d_out, e->geo.out.z, s);  // remaining planes
  } else {
    const float* w = e->p.mask_output_chunk ? inverse_weight(e, s) : nullptr;
    e->launches += finish_output(e, d_out, w, true, e->p.num_output_channels, vol(e->geo.out), s);
  }
  CFB_CUDA(cudaEventRecord(e->ev[3], s));
  e->timing_valid = true;
  return slab ? CFB_OK : output_range_status(e, s);
}

}  // namespace

extern "C" {

const char* cfb_last_error(void) { return g_last_error.c_str(); }
int cfb_version(void) { return 100; }

int cfb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int cfb_device_memory(int32_t device, int64_t* free_bytes, int64_t* total_bytes) {
  return guarded([&]() -> int {
    if (!free_bytes || !total_bytes) throw std::invalid_argument("null argument");
    if (cfb_device_count() <= 0) { set_last_error("no CUDA device available: chunkflow_b200 has no CPU fallback"); return CFB_ERR_CUDA; }
    CFB_CUDA(cudaSetDevice(device));
    size_t f = 0, t = 0;
    CFB_CUDA(cudaMemGetInfo(&f, &t));
    *free_bytes = (int64_t)f; *total_bytes = (int64_t)t;
    return CFB_OK;
  });
}

int cfb_create(const cfb_params* params, cfb_handle* out) {
  return guarded([&]() -> int {
    if (!params || !out) throw std::invalid_argument("null argument");
    if (params->struct_size != (int32_t)sizeof(cfb_params)) throw std::invalid_argument("cfb_params size mismatch (ABI)");
    const cfb_params& p = *params;
    if (p.framework != CFB_FRAMEWORK_UNET3L && p.framework != CFB_FRAMEWORK_IDENTITY) throw std::invalid_argument("unknown framework");
    if (p.num_input_channels != 1) throw std::invalid_argument("only one input channel is supported");
    if (p.num_output_channels < 1 || p.num_output_channels > 8) throw std::invalid_argument("num_output_channels must be in [1, 8]");
    if (p.augment != CFB_AUGMENT_NONE && p.augment != CFB_AUGMENT_REFERENCE && p.augment != CFB_AUGMENT_SPATIAL)
      throw std::invalid_argument("augment must be CFB_AUGMENT_NONE / _REFERENCE / _SPATIAL");
    if (p.augment && p.framework == CFB_FRAMEWORK_UNET3L && p.input_patch_size[1] != p.input_patch_size[2])
      throw std::invalid_argument("test-time augmentation transposes y and x: the patch must be square in y, x");
    auto e = std::make_unique<cfb_engine>();
    e->p = p;
    e->ip = Int3{p.input_patch_size[0], p.input_patch_size[1], p.input_patch_size[2]};
    e->op = Int3{p.output_patch_size[0], p.output_patch_size[1], p.output_patch_size[2]};
    e->ovl = Int3{p.output_patch_overlap[0], p.output_patch_overlap[1], p.output_patch_overlap[2]};
    e->ocm = Int3{p.output_crop_margin[0], p.output_crop_margin[1], p.output_crop_margin[2]};
    auto check3 = [](Int3 a, const char* what) {
      if (a.z <= 0 || a.y <= 0 || a.x <= 0) throw std::invalid_argument(std::string(what) + " must be positive");
    };
    check3(e->ip, "input_patch_size");
    check3(e->op, "output_patch_size");
    if (e->op.z > e->ip.z || e->op.y > e->ip.y || e->op.x > e->ip.x) throw std::invalid_argument("output patch larger than input patch");
    if ((e->ip.z - e->op.z) % 2 || (e->ip.y - e->op.y) % 2 || (e->ip.x - e->op.x) % 2) throw std::invalid_argument("input - output patch size must be even");
    if (e->ovl.z < 0 || e->ovl.y < 0 || e->ovl.x < 0 || e->ovl.z >= e->op.z || e->ovl.y >= e->op.y || e->ovl.x >= e->op.x)
      throw std::invalid_argument("output_patch_overlap must be in [0, output_patch_size)");
    if (e->ocm.z < 0 || e->ocm.y < 0 || e->ocm.x < 0) throw std::invalid_argument("negative output_crop_margin");
    // reference inferencer.py:109-122
    e->pcrop = Int3{(e->ip.z - e->op.z) / 2, (e->ip.y - e->op.y) / 2, (e->ip.x - e->op.x) / 2};
    e->ioverlap = Int3{2 * e->pcrop.z + e->ovl.z, 2 * e->pcrop.y + e->ovl.y, 2 * e->pcrop.x + e->ovl.x};
    e->istride = Int3{e->ip.z - e->ioverlap.z, e->ip.y - e->ioverlap.y, e->ip.x - e->ioverlap.x};
    if (p.framework == CFB_FRAMEWORK_UNET3L && (e->ip.y % 4 || e->ip.x % 4))
      throw std::invalid_argument("the 3-level U-Net pools (1,2,2) twice: patch y and x must be multiples of 4");
    if (e->ip.x % 4) throw std::invalid_argument("input patch x must be a multiple of 4");
    if (cfb_device_count() <= 0) { set_last_error("no CUDA device available: chunkflow_b200 has no CPU fallback"); return CFB_ERR_CUDA; }
    CFB_CUDA(cudaSetDevice(p.device));
    cudaDeviceProp prop;
    CFB_CUDA(cudaGetDeviceProperties(&prop, p.device));
    e->device_name = prop.name;
    if (prop.major != 9 || prop.minor != 0) {
      set_last_error(std::string("chunkflow_b200 kernels are built for sm_90a (H100) only; device is ") + prop.name);
      return CFB_ERR_CUDA;
    }
    e->h_mask = build_patch_mask(e->op, e->ovl);
    e->mask.grow(e->h_mask.size() * sizeof(float));
    CFB_CUDA(cudaMemcpy(e->mask.as(), e->h_mask.data(), e->h_mask.size() * sizeof(float), cudaMemcpyHostToDevice));
    e->flags.grow(2 * sizeof(unsigned int));
    CFB_CUDA(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
    CFB_CUDA(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    CFB_CUDA(cudaEventCreateWithFlags(&e->ev_ready, cudaEventDisableTiming));
    for (auto& ev : e->ev) CFB_CUDA(cudaEventCreate(&ev));
    e->net.configure(p.precision, e->ip, std::max(1, p.batch_size));
    *out = e.release();
    return CFB_OK;
  });
}

int cfb_destroy(cfb_handle h) {
  delete h;
  return CFB_OK;
}

const char* cfb_device_name(cfb_handle h) { return h ? h->device_name.c_str() : ""; }

int cfb_set_weight(cfb_handle h, const char* name, const float* host_data, int64_t numel) {
  return guarded([&]() -> int {
    if (!h || !name || !host_data || numel <= 0) throw std::invalid_argument("bad weight argument");
    h->host_w[name] = std::vector<float>(host_data, host_data + numel);
    return CFB_OK;
  });
}

int cfb_commit_weights(cfb_handle h) {
  return guarded([&]() -> int {
    if (!h) throw std::invalid_argument("null handle");
    CFB_CUDA(cudaSetDevice(h->p.device));
    std::string err;
    if (!h->net.load(h->host_w, h->p.num_output_channels, err)) {
      set_last_error(err);
      return CFB_ERR_WEIGHTS;
    }
    return CFB_OK;
  });
}

int cfb_patch_mask(cfb_handle h, float* host_out) {
  return guarded([&]() -> int {
    if (!h || !host_out) throw std::invalid_argument("null argument");
    std::memcpy(host_out, h->h_mask.data(), h->h_mask.size() * sizeof(float));
    return CFB_OK;
  });
}

int cfb_patch_grid(cfb_handle h, int64_t cz, int64_t cy, int64_t cx, int64_t* num_patches, int32_t* starts_zyx,
                   int64_t capacity) {
  return guarded([&]() -> int {
    if (!h || !num_patches) throw std::invalid_argument("null argument");
    const ChunkGeometry g = h->geometry(cz, cy, cx);
    *num_patches = (int64_t)g.z.in_start.size() * g.y.in_start.size() * g.x.in_start.size();
    if (starts_zyx) {
      int64_t k = 0;
      for (int a : g.z.in_start) for (int b : g.y.in_start) for (int c : g.x.in_start) {
        if (k >= capacity) return CFB_OK;
        starts_zyx[3 * k] = a; starts_zyx[3 * k + 1] = b; starts_zyx[3 * k + 2] = c; ++k;
      }
    }
    return CFB_OK;
  });
}

int cfb_output_shape(cfb_handle h, int64_t cz, int64_t cy, int64_t cx, int64_t out_czyx[4]) {
  return guarded([&]() -> int {
    if (!h || !out_czyx) throw std::invalid_argument("null argument");
    const Int3 out = h->geometry(cz, cy, cx).out;
    out_czyx[0] = h->p.num_output_channels;
    out_czyx[1] = out.z; out_czyx[2] = out.y; out_czyx[3] = out.x;
    return CFB_OK;
  });
}

int cfb_infer_chunk_device(cfb_handle h, const void* d_in, int32_t in_dtype, int64_t cz, int64_t cy, int64_t cx,
                           float* d_out, void* stream) {
  return guarded([&]() -> int {
    if (!h || !d_in || !d_out) throw std::invalid_argument("null argument");
    return infer_impl(h, d_in, in_dtype, cz, cy, cx, 0, 0, false, d_out, nullptr, (cudaStream_t)stream);
  });
}

int cfb_infer_slab_device(cfb_handle h, const void* d_in, int32_t in_dtype, int64_t cz, int64_t cy, int64_t cx,
                          int64_t zrow_begin, int64_t zrow_end, float* d_out, float* d_weight, void* stream) {
  return guarded([&]() -> int {
    if (!h || !d_in || !d_out) throw std::invalid_argument("null argument");
    return infer_impl(h, d_in, in_dtype, cz, cy, cx, zrow_begin, zrow_end, true, d_out, d_weight, (cudaStream_t)stream);
  });
}

int cfb_normalize_device(cfb_handle h, float* d_out, const float* d_weight, int32_t weight_is_inverse, int64_t channels,
                         int64_t oz, int64_t oy, int64_t ox, int32_t all_zero_input, void* stream) {
  return guarded([&]() -> int {
    if (!h || !d_out) throw std::invalid_argument("null argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    cudaStream_t s = (cudaStream_t)stream;
    // flags[0]: the nonzero flag the kernel reads (0 forces the output to zero, reference inferencer.py:387-393)
    const unsigned int init[2] = {all_zero_input ? 0u : 1u, 0u};
    CFB_CUDA(cudaMemcpyAsync(h->flags.as(), init, sizeof(init), cudaMemcpyHostToDevice, s));
    finish_output(h, d_out, d_weight, weight_is_inverse != 0, (int)channels, oz * oy * ox, s);
    return output_range_status(h, s);
  });
}

int cfb_slab_nonzero(cfb_handle h, int32_t* nonzero, void* stream) {
  return guarded([&]() -> int {
    if (!h || !nonzero) throw std::invalid_argument("null argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    unsigned int flag = 0;
    CFB_CUDA(cudaMemcpyAsync(&flag, h->flags.as(), sizeof(flag), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CFB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    *nonzero = flag != 0u;
    return CFB_OK;
  });
}

int cfb_halo_add_device(float* d_dst, const float* d_src, int64_t count, void* stream) {
  return guarded([&]() -> int {
    if (!d_dst || !d_src || count < 0) throw std::invalid_argument("bad argument");
    launch_halo_add(d_dst, d_src, count, (cudaStream_t)stream);
    return CFB_OK;
  });
}

int cfb_weight_volume_device(cfb_handle h, int64_t cz, int64_t cy, int64_t cx, int64_t z_begin, int64_t z_end, int32_t invert,
                             float* d_weight, void* stream) {
  return guarded([&]() -> int {
    if (!h || !d_weight) throw std::invalid_argument("null argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    cudaStream_t s = (cudaStream_t)stream;
    const ChunkGeometry g = h->geometry(cz, cy, cx);
    if (z_begin < 0 || z_end > g.out.z || z_begin > z_end) throw std::invalid_argument("bad plane range");
    DeviceBuffer tables;
    launch_weight_volume(h->mask.as<float>(), h->op, upload_cover_tables(g, h->op, tables, s), g.out, d_weight, invert != 0, s,
                         (int)z_begin, (int)z_end);
    CFB_CUDA(cudaStreamSynchronize(s));  // the tables are a temporary
    return CFB_OK;
  });
}

int cfb_infer_chunk_host(cfb_handle h, const void* h_in, int32_t in_dtype, int64_t cz, int64_t cy, int64_t cx,
                         float* h_out) {
  return guarded([&]() -> int {
    if (!h || !h_in || !h_out) throw std::invalid_argument("null argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    int64_t shape[4];
    int rc = cfb_output_shape(h, cz, cy, cx, shape);
    if (rc != CFB_OK) return rc;
    const size_t in_bytes = (size_t)cz * cy * cx * (in_dtype == CFB_DTYPE_U8 ? 1 : 4);
    const size_t out_bytes = (size_t)shape[0] * shape[1] * shape[2] * shape[3] * sizeof(float);
    h->host_in.grow(in_bytes);
    h->host_out.grow(out_bytes);
    void* d_in = h->host_in.as();
    float* d_out = h->host_out.as<float>();
    cudaStream_t s = h->own_stream;
    // host arrays in pageable memory (what a drop-in caller has: plain numpy) move through the engine's own pinned ring,
    // copied by host threads; CFB_NO_HOST_STAGING=1 leaves the staging to the driver
    static const bool no_staging = getenv("CFB_NO_HOST_STAGING") != nullptr;
    CFB_CUDA(cudaEventRecord(h->ev[4], s));
    if (!no_staging && in_bytes >= ((size_t)64 << 20) && !is_pinned_host(h_in)) {
      if (!h->stager) h->stager = std::make_unique<HostStager>(h->p.device);
      h->stager->upload(h_in, d_in, in_bytes, s);
    } else {
      CFB_CUDA(cudaMemcpyAsync(d_in, h_in, in_bytes, cudaMemcpyHostToDevice, s));
    }
    CFB_CUDA(cudaEventRecord(h->ev[5], s));
    Progressive pg;
    pg.h_out = h_out;
    pg.copy_stream = h->copy_stream;
    pg.ready = h->ev_ready;
    if (!no_staging && out_bytes >= ((size_t)8 << 20) && !is_pinned_host(h_out)) {
      if (!h->stager) h->stager = std::make_unique<HostStager>(h->p.device);
      pg.stager = h->stager.get();
    }
    const bool progressive = !h->p.has_myelin_threshold;
    rc = infer_impl(h, d_in, in_dtype, cz, cy, cx, 0, 0, false, d_out, nullptr, s, progressive ? &pg : nullptr);
    if (rc != CFB_OK) {
      cudaStreamSynchronize(h->copy_stream);
      if (pg.stager) { try { pg.stager->drain(); } catch (...) {} }
      return rc;
    }
    CFB_CUDA(cudaEventRecord(h->ev[6], s));
    if (!progressive) {
      if (pg.stager) pg.stager->push(d_out, h_out, out_bytes, s, h->copy_stream);
      else CFB_CUDA(cudaMemcpyAsync(h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, s));
    }
    CFB_CUDA(cudaEventRecord(h->ev[7], s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (pg.stager) pg.stager->drain();
    CFB_CUDA(cudaStreamSynchronize(h->copy_stream));
    return CFB_OK;
  });
}

int cfb_patch_forward_host(cfb_handle h, const float* h_patches, int32_t batch, float* h_out) {
  return guarded([&]() -> int {
    if (!h || !h_patches || !h_out || batch <= 0) throw std::invalid_argument("bad argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    if (h->p.framework == CFB_FRAMEWORK_UNET3L && !h->net.ready()) { set_last_error("weights not committed"); return CFB_ERR_WEIGHTS; }
    cudaStream_t s = h->own_stream;
    const int C = h->p.num_output_channels;
    const int64_t in_vol = vol(h->ip), out_vol = vol(h->op);
    h->plugin_out.grow((size_t)batch * C * out_vol * sizeof(float));
    const int B = std::max(1, h->p.batch_size);
    for (int i = 0; i < batch; i += B) {
      const int nb = std::min(B, batch - i);
      float* dst = h->plugin_out.as<float>() + (int64_t)i * C * out_vol;
      if (h->p.framework == CFB_FRAMEWORK_IDENTITY) {
        float* stage = h->net.patch_input_buffer(nb);
        CFB_CUDA(cudaMemcpyAsync(stage, h_patches + (int64_t)i * in_vol, (size_t)nb * in_vol * sizeof(float), cudaMemcpyHostToDevice, s));
        launch_crop_mask(stage, 1, h->ip, h->op, h->pcrop, h->mask.as<float>(), nb, dst, C, /*repeat=*/true, s);
      } else {
        h->net.forward_from_host_patches(h_patches + (int64_t)i * in_vol, nb, s);
        h->net.crop_mask(h->op, h->pcrop, h->mask.as<float>(), nb, dst, C, s);
      }
    }
    CFB_CUDA(cudaMemcpyAsync(h_out, h->plugin_out.as(), (size_t)batch * C * out_vol * sizeof(float), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    return CFB_OK;
  });
}

int cfb_make_patch_mask(const int32_t patch_size[3], const int32_t overlap[3], float* host_out) {
  return guarded([&]() -> int {
    if (!patch_size || !overlap || !host_out) throw std::invalid_argument("null argument");
    const Int3 p{patch_size[0], patch_size[1], patch_size[2]}, o{overlap[0], overlap[1], overlap[2]};
    if (p.z <= 0 || p.y <= 0 || p.x <= 0 || o.z < 0 || o.y < 0 || o.x < 0 || o.z >= p.z || o.y >= p.y || o.x >= p.x)
      throw std::invalid_argument("bad patch size / overlap");
    std::vector<float> m = build_patch_mask(p, o);
    std::memcpy(host_out, m.data(), m.size() * sizeof(float));
    return CFB_OK;
  });
}

int cfb_plugin_begin(cfb_handle h, const void* h_in, int32_t in_dtype, int64_t cz, int64_t cy, int64_t cx) {
  return guarded([&]() -> int {
    if (!h || !h_in) throw std::invalid_argument("null argument");
    if (in_dtype != CFB_DTYPE_U8 && in_dtype != CFB_DTYPE_F32) throw std::invalid_argument("unsupported input dtype");
    CFB_CUDA(cudaSetDevice(h->p.device));
    cudaStream_t s = h->own_stream;
    prepare_chunk(h, cz, cy, cx, s);
    const size_t in_bytes = (size_t)cz * cy * cx * (in_dtype == CFB_DTYPE_U8 ? 1 : 4);
    h->host_in.grow(in_bytes);
    h->host_out.grow((size_t)h->p.num_output_channels * vol(h->geo.out) * sizeof(float));
    CFB_CUDA(cudaMemcpyAsync(h->host_in.as(), h_in, in_bytes, cudaMemcpyHostToDevice, s));
    start_chunk(h, h->host_in.as(), in_dtype, h->host_out.as<float>(), s);
    h->plugin_dtype = in_dtype;
    h->plugin_active = true;
    return CFB_OK;
  });
}

int cfb_plugin_extract(cfb_handle h, int64_t first, int32_t nb, float* h_patches) {
  return guarded([&]() -> int {
    if (!h || !h_patches || !h->plugin_active) throw std::invalid_argument("cfb_plugin_begin was not called");
    if (first < 0 || nb <= 0 || first + nb > (int64_t)h->h_patches.size()) throw std::invalid_argument("patch range out of bounds");
    CFB_CUDA(cudaSetDevice(h->p.device));
    cudaStream_t s = h->own_stream;
    const size_t bytes = (size_t)nb * vol(h->ip) * sizeof(float);
    h->plugin_in.grow(bytes);
    launch_extract_patches(h->host_in.as(), h->plugin_dtype, h->geo.size, h->patches.as<PatchPos>() + first, nb, h->ip,
                           h->plugin_in.as<float>(), s);
    CFB_CUDA(cudaMemcpyAsync(h_patches, h->plugin_in.as(), bytes, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    return CFB_OK;
  });
}

int cfb_plugin_blend(cfb_handle h, int64_t first, int32_t nb, const float* h_masked_outputs) {
  return guarded([&]() -> int {
    if (!h || !h_masked_outputs || !h->plugin_active) throw std::invalid_argument("cfb_plugin_begin was not called");
    if (first < 0 || nb <= 0 || first + nb > (int64_t)h->h_patches.size()) throw std::invalid_argument("patch range out of bounds");
    CFB_CUDA(cudaSetDevice(h->p.device));
    cudaStream_t s = h->own_stream;
    const int C = h->p.num_output_channels;
    const size_t bytes = (size_t)nb * C * vol(h->op) * sizeof(float);
    h->plugin_out.grow(bytes);
    CFB_CUDA(cudaMemcpyAsync(h->plugin_out.as(), h_masked_outputs, bytes, cudaMemcpyHostToDevice, s));
    // already cropped and masked by the plugin: crop 0, no mask
    launch_blend_patches(h->plugin_out.as<float>(), C, h->op, h->op, Int3{0, 0, 0}, nullptr, h->patches.as<PatchPos>() + first, nb,
                         h->host_out.as<float>(), C, h->geo.out, 1.0f, s);
    CFB_CUDA(cudaStreamSynchronize(s));  // the caller may reuse its host buffer
    return CFB_OK;
  });
}

int cfb_plugin_end(cfb_handle h, float* h_out) {
  return guarded([&]() -> int {
    if (!h || !h_out || !h->plugin_active) throw std::invalid_argument("cfb_plugin_begin was not called");
    CFB_CUDA(cudaSetDevice(h->p.device));
    cudaStream_t s = h->own_stream;
    h->plugin_active = false;
    const int C = h->p.num_output_channels;
    const int64_t nvox = vol(h->geo.out);
    float* out = h->host_out.as<float>();
    const float* w = h->p.mask_output_chunk ? inverse_weight(h, s) : nullptr;
    finish_output(h, out, w, true, C, nvox, s);
    CFB_CUDA(cudaMemcpyAsync(h_out, out, (size_t)C * nvox * sizeof(float), cudaMemcpyDeviceToHost, s));
    const int rc = output_range_status(h, s);
    CFB_CUDA(cudaStreamSynchronize(s));
    return rc;
  });
}

int cfb_last_timing(cfb_handle h, float ms[5], int64_t* launches) {
  return guarded([&]() -> int {
    if (!h || !ms) throw std::invalid_argument("null argument");
    for (int i = 0; i < 5; ++i) ms[i] = 0.f;
    if (launches) *launches = h->launches;
    if (!h->timing_valid) return CFB_OK;
    CFB_CUDA(cudaSetDevice(h->p.device));
    CFB_CUDA(cudaEventSynchronize(h->ev[3]));
    CFB_CUDA(cudaEventElapsedTime(&ms[0], h->ev[0], h->ev[3]));
    CFB_CUDA(cudaEventElapsedTime(&ms[1], h->ev[1], h->ev[2]));
    CFB_CUDA(cudaEventElapsedTime(&ms[2], h->ev[2], h->ev[3]));
    if (cudaEventQuery(h->ev[7]) == cudaSuccess && cudaEventQuery(h->ev[4]) == cudaSuccess) {
      if (cudaEventElapsedTime(&ms[3], h->ev[4], h->ev[5]) != cudaSuccess) ms[3] = 0.f;
      if (cudaEventElapsedTime(&ms[4], h->ev[6], h->ev[7]) != cudaSuccess) ms[4] = 0.f;
    }
    cudaGetLastError();
    return CFB_OK;
  });
}

int cfb_set_profiling(cfb_handle h, int32_t enabled) {
  return guarded([&]() -> int {
    if (!h) throw std::invalid_argument("null handle");
    CFB_CUDA(cudaSetDevice(h->p.device));
    h->net.set_profiling(enabled != 0);
    return CFB_OK;
  });
}

int cfb_layer_timing(cfb_handle h, int32_t capacity, int32_t* count, char (*names)[32], float* ms, int64_t* launches) {
  return guarded([&]() -> int {
    if (!h || !count || !names || !ms || !launches) throw std::invalid_argument("null argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    std::vector<std::string> n; std::vector<float> m; std::vector<int64_t> l;
    h->net.layer_timing(n, m, l);
    *count = (int32_t)std::min<size_t>(n.size(), (size_t)capacity);
    for (int i = 0; i < *count; ++i) {
      std::strncpy(names[i], n[i].c_str(), 31); names[i][31] = 0;
      ms[i] = m[i]; launches[i] = l[i];
    }
    return CFB_OK;
  });
}

int cfb_debug_net_forward_host(cfb_handle h, const float* h_patch, float* h_out) {
  return guarded([&]() -> int {
    if (!h || !h_patch || !h_out) throw std::invalid_argument("null argument");
    CFB_CUDA(cudaSetDevice(h->p.device));
    if (!h->net.ready()) { set_last_error("weights not committed"); return CFB_ERR_WEIGHTS; }
    cudaStream_t s = h->own_stream;
    h->net.forward_from_host_patches(h_patch, 1, s);
    h->net.copy_raw_output_to_host(h_out, s);
    CFB_CUDA(cudaStreamSynchronize(s));
    return CFB_OK;
  });
}

int cfb_debug_layer_host(cfb_handle h, const cfb_layer_args* args) {
  return guarded([&]() -> int {
    if (!h || !args) throw std::invalid_argument("null argument");
    if (args->struct_size != (int32_t)sizeof(cfb_layer_args)) throw std::invalid_argument("cfb_layer_args size mismatch");
    CFB_CUDA(cudaSetDevice(h->p.device));
    return h->net.debug_layer(*args, h->own_stream);
  });
}

}  // extern "C"
