// `skeletonize` (reference chunkflow/plugins/skeletonize.py -> kimimaro.skeletonize): a TEASAR skeleton of every object of a
// segmentation chunk, restated in oracle/skeleton_oracle.py (kimimaro is not vendored: its skeletons are not reproduced).  On the
// device (skeleton_kernels.cuh):
//   count     the multi-label distance to the boundary (x run pass, y and z Felzenszwalb-Huttenlocher passes); 26-connected
//             components by union-find (union_find.cuh); the kept components numbered in raster order of their first voxel
//   skeleton  roots (one atomicMax per voxel), the geodesic field D by block-tiled relaxation until a sweep changes nothing, the
//             parents, one stable sort of every object's voxels by (object, D descending, index) (radix_sort.cuh), then rounds:
//             one thread per object moves a cursor past invalidated voxels to its target and traces it, and the invalidation
//             balls are spread over the GPU.  Only a "found a target" flag comes to the host between rounds.
//   read      the skeleton voxels grouped by id on the host: vertices, edges and radii per label.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <stdexcept>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

constexpr int kSkThreads = 256;
constexpr int kMcThreads = kSkThreads;   // radix_sort.cuh
constexpr int kSkStats = 8;              // cfb_skeleton_device's stats

#include "union_find.cuh"
#include "raster_scan.cuh"
#include "radix_sort.cuh"
#include "skeleton_kernels.cuh"

int sk_grid(int64_t work) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(work, kSkThreads), 132 * 16)); }

SkGeom sk_geom(int64_t z, int64_t y, int64_t x, const double* voxel_size) {
  if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX)
    throw std::invalid_argument("skeletonize: every axis of the chunk has 1 to 2^31 - 1 voxels");
  if (z * y > ((int64_t)1 << 62) / x || z * y * x >= ((int64_t)1 << 32))
    throw std::invalid_argument("skeletonize: the chunk must have fewer than 2^32 voxels");
  if (!voxel_size) throw std::invalid_argument("skeletonize: null voxel size");
  SkGeom g;
  g.Z = z; g.Y = y; g.X = x;
  g.n = z * y * x;
  for (int a = 0; a < 3; ++a) {
    if (!(std::isfinite(voxel_size[a]) && voxel_size[a] > 0.0))
      throw std::invalid_argument("skeletonize: the voxel size is three positive finite numbers");
    g.w[a] = voxel_size[a];
  }
  for (int k = 0; k < 27; ++k) {   // summed z, y, x, each square rounded on its own (the oracle's step_length)
    const double a = (double)std::abs(k / 9 - 1) * g.w[0], b = (double)std::abs((k / 3) % 3 - 1) * g.w[1],
                 c = (double)std::abs(k % 3 - 1) * g.w[2];
    const double aa = a * a, bb = b * b, cc = c * c;
    g.len[k] = std::sqrt((aa + bb) + cc);
  }
  return g;
}

// D must stay finite and every step must raise it, so that every Parent chain ends at the root (DESIGN.md f10): a path has
// fewer than `n` steps, each costing at most the diagonal step times PDRF <= pdrf_scale + 1; below 2^53 times the smallest
// voxel size, half an ulp of D is less than the cheapest step.  The same expression, rounded the same way, in
// oracle/skeleton_oracle.py and chunkflow_b200/flow/skeleton.py.
void sk_check_geodesic(const SkGeom& g, double pdrf_scale) {
  const double min_w = std::min(g.w[0], std::min(g.w[1], g.w[2]));
  const double bound = (((pdrf_scale + 1.0) * g.len[0]) * (double)g.n) * (1.0 + 0x1p-19);
  if (!(std::isfinite(g.len[0]) && bound < 0x1p53 * min_w))
    throw std::invalid_argument("skeletonize: D must stay finite and strictly increasing: (pdrf_scale + 1) * diagonal step * chunk "
                                "voxels * (1 + 2^-19) must be below 2^53 * the smallest voxel size");
}

SkTiles sk_tiles(const SkGeom& g) {
  SkTiles t;
  t.t[0] = ceil_div64(g.Z, kSkTile); t.t[1] = ceil_div64(g.Y, kSkTile); t.t[2] = ceil_div64(g.X, kSkTile);
  t.count = t.t[0] * t.t[1] * t.t[2];
  return t;
}

// workspace of the distance transform alone: the y pass's squared distances (n x 8 B) | the x pass (n x 4 B) | the envelope
// stacks (n x 4 B)
struct SkEdtWork {
  double* d2;
  uint32_t *kx, *vstack;
  int64_t bytes;
};

SkEdtWork sk_edt_work(void* base, const SkGeom& g) {
  SkEdtWork e;
  e.d2 = static_cast<double*>(base);
  e.kx = reinterpret_cast<uint32_t*>(e.d2 + g.n);
  e.vstack = e.kx + g.n;
  e.bytes = 16 * g.n;
  return e;
}

// workspace of a skeleton (8-byte words first):
//   stats (8 x 8 B: kept voxels, objects, the relaxation's change flag, "used by cfb_skeleton_device") | D (n x 8 B) | component
//   counts, then Parent (n x 4 B) | root flags and ranks, then the sort positions | DBF | union-find parents | objects | tile flags
//   (2 x tiles) | scan sums | valid, on-skeleton (n x 1 B).  D, the counts and the ranks are the distance transform's workspace
//   (sk_edt_work) while it runs.
struct SkWork {
  unsigned long long* stats;
  double* D;
  float* dbf;
  uint32_t *P, *obj, *count, *rank, *dirty, *next, *sums;
  uint8_t *valid, *on;
  int64_t bytes;
};

SkWork sk_work(void* base, const SkGeom& g) {
  SkWork w;
  const int64_t n = g.n, tiles = sk_tiles(g).count;
  w.stats = static_cast<unsigned long long*>(base);
  w.D = reinterpret_cast<double*>(w.stats + 8);
  w.count = reinterpret_cast<uint32_t*>(w.D + n);
  w.rank = w.count + n;
  w.dbf = reinterpret_cast<float*>(w.rank + n);
  w.P = reinterpret_cast<uint32_t*>(w.dbf + n);
  w.obj = w.P + n;
  w.dirty = w.obj + n;
  w.next = w.dirty + tiles;
  w.sums = w.next + tiles;
  w.valid = reinterpret_cast<uint8_t*>(w.sums + mc_chunks(n) + 1);
  w.on = w.valid + n;
  w.bytes = (int64_t)((char*)(w.on + n) - (char*)base);
  return w;
}

// buffer of K objects with m voxels in all (8-byte words first):
//   sort ids, values and their copies (4 m x 8 B) | root keys (K x 8 B) | round counters (kSkCounters x 8 B) | object starts (K + 1) |
//   cursors (K) | bounding boxes (6 K) | path voxels (m) | radix histograms (256 chunks(m)) | scan sums (x 4 B)
struct SkBuffer {
  unsigned long long *ids, *vals, *ids2, *vals2, *key, *counters;
  uint32_t *start, *cursor, *path, *hist, *sums;
  int* bbox;
  int64_t bytes;
};

SkBuffer sk_buffer(void* base, int64_t K, int64_t m) {
  SkBuffer b;
  unsigned long long* w = static_cast<unsigned long long*>(base);
  b.ids = w; b.vals = w + m; b.ids2 = w + 2 * m; b.vals2 = w + 3 * m;
  b.key = w + 4 * m;
  b.counters = b.key + K;
  uint32_t* u = reinterpret_cast<uint32_t*>(b.counters + kSkCounters);
  b.start = u;
  b.cursor = b.start + K + 1;
  b.bbox = reinterpret_cast<int*>(b.cursor + K);
  b.path = reinterpret_cast<uint32_t*>(b.bbox + 6 * K);
  b.hist = b.path + m;
  const int64_t hist_len = 256 * mc_chunks(m);
  b.sums = b.hist + hist_len;
  b.bytes = (int64_t)((char*)(b.sums + mc_chunks(std::max(hist_len, std::max(m, K + 1))) + 1) - (char*)base);
  return b;
}

void sk_check_labels(const void* d_labels, int32_t dtype) {
  if (!d_labels) throw std::invalid_argument("skeletonize: null segmentation");
  if (dtype != CFB_DTYPE_U32 && dtype != CFB_DTYPE_U64) throw std::invalid_argument("skeletonize: the ids are uint32 or uint64");
}

template <typename T>
void sk_edt(const T* seg, const SkGeom& g, const SkEdtWork& e, float* dbf, cudaStream_t s) {
  launch(sk_edt_x_kernel<T>, (unsigned)std::min<int64_t>(ceil_div64(g.Z * g.Y, kSkRows), 132 * 32), kSkRows, 0, s, seg, g, e.kx);
  launch(sk_edt_col_kernel<T, false>, sk_grid(g.Z * g.X), kSkThreads, 0, s, seg, g, (const uint32_t*)e.kx, e.d2, e.vstack, dbf);
  launch(sk_edt_col_kernel<T, true>, sk_grid(g.Y * g.X), kSkThreads, 0, s, seg, g, (const uint32_t*)e.kx, e.d2, e.vstack, dbf);
}

template <typename T>
void sk_count(const T* seg, const SkGeom& g, const unsigned long long* skip, int64_t num_skip, uint64_t dust, const SkWork& w,
              cudaStream_t s) {
  sk_edt(seg, g, sk_edt_work(w.D, g), w.dbf, s);
  const Int3 sz{(int)g.Z, (int)g.Y, (int)g.X};
  launch(sk_init_kernel, sk_grid(g.n), kSkThreads, 0, s, w.P, w.count, g.n);
  launch(cc_merge_kernel<T>, sk_grid(g.n), kSkThreads, 0, s, seg, w.P, sz, 13);
  launch(sk_flatten_kernel<T>, sk_grid(g.n), kSkThreads, 0, s, seg, w.P, w.count, g.n);
  launch(sk_root_flags_kernel<T>, sk_grid(g.n), kSkThreads, 0, s, seg, (const uint32_t*)w.P, (const uint32_t*)w.count, skip, num_skip, dust,
         g.n, w.rank, w.stats);
  const uint32_t objects = mc_scan(w.rank, g.n, w.sums, s);
  CFB_CUDA(cudaMemcpyAsync(w.stats + 1, &objects, 4, cudaMemcpyHostToDevice, s));
  launch(sk_objects_kernel<T>, sk_grid(g.n), kSkThreads, 0, s, seg, (const uint32_t*)w.P, (const uint32_t*)w.count, skip, num_skip, dust,
         (const uint32_t*)w.rank, g.n, w.obj);
}

template <typename T>
void sk_gather(const T* seg, const SkBuffer& b, int64_t S, const SkWork& w, cudaStream_t s) {
  launch(sk_gather_kernel<T>, sk_grid(S), kSkThreads, 0, s, seg, (const uint32_t*)b.path, S, (const float*)w.dbf,
         (const uint32_t*)w.count, b.ids, b.vals);
}

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_skeleton_workspace(int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    if (!workspace_bytes) throw std::invalid_argument("skeletonize: null output");
    const double unit[3] = {1.0, 1.0, 1.0};
    *workspace_bytes = sk_work(nullptr, sk_geom(z, y, x, unit)).bytes;
    return CFB_OK;
  });
}

extern "C" int cfb_edt_workspace(int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    if (!workspace_bytes) throw std::invalid_argument("distance transform: null output");
    const double unit[3] = {1.0, 1.0, 1.0};
    *workspace_bytes = sk_edt_work(nullptr, sk_geom(z, y, x, unit)).bytes;
    return CFB_OK;
  });
}

extern "C" int cfb_edt_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const double* voxel_size, float* d_dbf,
                              void* d_workspace, void* stream) {
  return guarded([&]() -> int {
    sk_check_labels(d_labels, dtype);
    if (!d_dbf || !d_workspace) throw std::invalid_argument("distance transform: null argument");
    const SkGeom g = sk_geom(z, y, x, voxel_size);
    const SkEdtWork e = sk_edt_work(d_workspace, g);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == CFB_DTYPE_U32) sk_edt((const uint32_t*)d_labels, g, e, d_dbf, s);
    else sk_edt((const uint64_t*)d_labels, g, e, d_dbf, s);
    return CFB_OK;
  });
}

extern "C" int cfb_skeleton_count_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const double* voxel_size,
                                         const uint64_t* d_skip_ids, int64_t num_skip, int64_t dust_threshold, void* d_workspace,
                                         int64_t* num_objects, int64_t* num_voxels, int64_t* buffer_bytes, void* stream) {
  return guarded([&]() -> int {
    sk_check_labels(d_labels, dtype);
    if (!d_workspace || !num_objects || !num_voxels || !buffer_bytes) throw std::invalid_argument("skeletonize: null argument");
    if (num_skip < 0 || (num_skip > 0 && !d_skip_ids)) throw std::invalid_argument("skeletonize: bad skip list");
    if (dust_threshold < 0) throw std::invalid_argument("skeletonize: dust_threshold is >= 0");
    const SkGeom g = sk_geom(z, y, x, voxel_size);
    const SkWork w = sk_work(d_workspace, g);
    cudaStream_t s = (cudaStream_t)stream;
    CFB_CUDA(cudaMemsetAsync(w.stats, 0, 8 * 8, s));
    const unsigned long long* skip = (const unsigned long long*)d_skip_ids;
    if (dtype == CFB_DTYPE_U32) sk_count((const uint32_t*)d_labels, g, skip, num_skip, (uint64_t)dust_threshold, w, s);
    else sk_count((const uint64_t*)d_labels, g, skip, num_skip, (uint64_t)dust_threshold, w, s);
    unsigned long long h[2];
    CFB_CUDA(cudaMemcpyAsync(h, w.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_voxels = (int64_t)h[0];
    *num_objects = (int64_t)(uint32_t)h[1];
    *buffer_bytes = sk_buffer(nullptr, *num_objects, *num_voxels).bytes;
    return CFB_OK;
  });
}

extern "C" int cfb_skeleton_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const double* voxel_size,
                                   const double* params, int32_t pdrf_exponent, void* d_workspace, int64_t num_objects, int64_t num_voxels,
                                   void* d_buffer, int64_t buffer_bytes, int64_t* num_skeleton_voxels, double* stats, void* stream) {
  return guarded([&]() -> int {
    sk_check_labels(d_labels, dtype);
    if (!params || !d_workspace || !num_skeleton_voxels) throw std::invalid_argument("skeletonize: null argument");
    SkParams prm{params[0], params[1], params[2], pdrf_exponent};
    for (int k = 0; k < 3; ++k)
      if (!(std::isfinite(params[k]) && params[k] >= 0.0)) throw std::invalid_argument("skeletonize: scale, const and pdrf_scale are finite and >= 0");
    if (pdrf_exponent < 1 || pdrf_exponent > 16) throw std::invalid_argument("skeletonize: pdrf_exponent is an integer from 1 to 16");
    const SkGeom g = sk_geom(z, y, x, voxel_size);
    sk_check_geodesic(g, prm.pdrf_scale);
    const SkWork w = sk_work(d_workspace, g);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long h[4];
    CFB_CUDA(cudaMemcpyAsync(h, w.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if ((int64_t)h[0] != num_voxels || (int64_t)(uint32_t)h[1] != num_objects)
      throw std::invalid_argument("skeletonize: the counts are not those of cfb_skeleton_count_device for this workspace");
    if (h[3]) throw std::invalid_argument("skeletonize: one cfb_skeleton_device per cfb_skeleton_count_device (it overwrites the counts)");
    const unsigned long long used = 1ULL;
    CFB_CUDA(cudaMemcpyAsync(w.stats + 3, &used, 8, cudaMemcpyHostToDevice, s));
    const int64_t K = num_objects, m = num_voxels;
    double st[kSkStats] = {};   // sweeps, rounds, paths, skeleton voxels, relaxation ms, sort ms, rounds ms, trace ms
    *num_skeleton_voxels = 0;
    if (K == 0) {
      if (stats) std::memcpy(stats, st, sizeof(st));
      return CFB_OK;
    }
    if (!d_buffer) throw std::invalid_argument("skeletonize: null buffer");
    const SkBuffer b = sk_buffer(d_buffer, K, m);
    if (buffer_bytes < b.bytes) throw std::invalid_argument("skeletonize: the buffer is smaller than cfb_skeleton_count_device asked for");
    // objects: starts, roots, bounding boxes
    CFB_CUDA(cudaMemsetAsync(b.start, 0, (size_t)(K + 1) * 4, s));
    launch(sk_object_init_kernel, sk_grid(g.n), kSkThreads, 0, s, (const uint32_t*)w.P, (const uint32_t*)w.obj, (const uint32_t*)w.count,
           g.n, b.start, b.key, b.bbox, K);
    if ((int64_t)mc_scan(b.start, K + 1, b.sums, s) != m) throw std::runtime_error("skeletonize: the objects do not hold the counted voxels");
    launch(sk_roots_kernel, sk_grid(g.n), kSkThreads, 0, s, (const uint32_t*)w.obj, (const float*)w.dbf, g, b.key, b.bbox);
    // D: block-tiled relaxation, sweeps until one changes nothing
    const auto t0 = std::chrono::steady_clock::now();
    const SkTiles tl = sk_tiles(g);
    uint32_t* changed = reinterpret_cast<uint32_t*>(w.stats + 2);
    uint32_t *dirty = w.dirty, *next = w.next;
    launch(sk_d_init_kernel, sk_grid(g.n), kSkThreads, 0, s, w.D, g.n);
    CFB_CUDA(cudaMemsetAsync(dirty, 0, (size_t)tl.count * 4, s));
    launch(sk_d_roots_kernel, sk_grid(K), kSkThreads, 0, s, (const unsigned long long*)b.key, K, g, tl, w.D, dirty);
    for (;;) {
      CFB_CUDA(cudaMemsetAsync(next, 0, (size_t)tl.count * 4, s));
      CFB_CUDA(cudaMemsetAsync(changed, 0, 4, s));
      launch(sk_relax_kernel, (unsigned)std::min<int64_t>(tl.count, 132 * 8), kSkThreads, 0, s, (const uint32_t*)w.obj, (const float*)w.dbf, g,
             prm, (const unsigned long long*)b.key, tl, w.D, (const uint32_t*)dirty, next, changed);
      uint32_t c = 0;
      CFB_CUDA(cudaMemcpyAsync(&c, changed, 4, cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaStreamSynchronize(s));
      st[0] += 1;
      if (!c) break;
      std::swap(dirty, next);
    }
    launch(sk_parent_kernel, sk_grid(g.n), kSkThreads, 0, s, (const uint32_t*)w.obj, (const float*)w.dbf, g, prm,
           (const unsigned long long*)b.key, (const double*)w.D, w.count);
    CFB_CUDA(cudaStreamSynchronize(s));
    st[4] = ms_since(t0);
    // every object's voxels by (object, D descending, index): a stable sort by ~D bits, then by object
    const auto t1 = std::chrono::steady_clock::now();
    launch(sk_flag_kernel, sk_grid(g.n), kSkThreads, 0, s, (const uint32_t*)w.obj, g.n, w.rank);
    if ((int64_t)mc_scan(w.rank, g.n, w.sums, s) != m) throw std::runtime_error("skeletonize: the voxels of the objects changed");
    launch(sk_emit_kernel, sk_grid(g.n), kSkThreads, 0, s, (const uint32_t*)w.obj, (const double*)w.D, (const uint32_t*)w.rank, g.n,
           b.ids, b.vals);
    mc_sort(b.ids, b.vals, b.ids2, b.vals2, m, 64, b.hist, b.sums, s);
    launch(sk_object_keys_kernel, sk_grid(m), kSkThreads, 0, s, (const uint32_t*)w.obj, (const unsigned long long*)b.vals, m, b.ids);
    mc_sort(b.ids, b.vals, b.ids2, b.vals2, m, 32, b.hist, b.sums, s);
    CFB_CUDA(cudaStreamSynchronize(s));
    st[5] = ms_since(t1);
    // rounds; the trace is timed on its own (it starts on an idle stream and ends in a synchronise)
    const auto t2 = std::chrono::steady_clock::now();
    CFB_CUDA(cudaMemsetAsync(w.valid, 1, (size_t)g.n, s));
    CFB_CUDA(cudaMemsetAsync(w.on, 0, (size_t)g.n, s));
    CFB_CUDA(cudaMemcpyAsync(b.cursor, b.start, (size_t)K * 4, cudaMemcpyDeviceToDevice, s));
    CFB_CUDA(cudaMemsetAsync(b.counters, 0, kSkCounters * 8, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    for (;;) {
      const auto t3 = std::chrono::steady_clock::now();
      launch(sk_round_begin_kernel, 1, 1, 0, s, b.counters);
      launch(sk_trace_kernel, sk_grid(K), kSkThreads, 0, s, (const unsigned long long*)b.vals, (const uint32_t*)b.start, b.cursor, K,
             (const uint8_t*)w.valid, (const uint32_t*)w.count, w.on, b.path, b.counters);
      CFB_CUDA(cudaStreamSynchronize(s));
      st[7] += ms_since(t3);
      launch(sk_invalidate_kernel, dim3(264, 16), kSkThreads, 0, s, (const uint32_t*)b.path, (const unsigned long long*)b.counters,
             (const uint32_t*)w.obj, (const float*)w.dbf, g, prm, (const int*)b.bbox, w.valid);
      unsigned long long flags[3] = {0, 0, 0};   // found a target, paths, broken chain
      CFB_CUDA(cudaMemcpyAsync(flags, b.counters + 2, sizeof(flags), cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaStreamSynchronize(s));
      if (flags[2]) throw std::runtime_error("skeletonize: a Parent chain does not end at its root (D is not strictly increasing)");
      if (!flags[0]) break;
      st[1] += 1;
    }
    unsigned long long c[4];
    CFB_CUDA(cudaMemcpyAsync(c, b.counters, sizeof(c), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    st[6] = ms_since(t2);
    st[2] = (double)c[3];
    st[3] = (double)c[0];
    const int64_t S = (int64_t)c[0];
    if (S > m) throw std::runtime_error("skeletonize: more skeleton voxels than object voxels");
    if (dtype == CFB_DTYPE_U32) sk_gather((const uint32_t*)d_labels, b, S, w, s);
    else sk_gather((const uint64_t*)d_labels, b, S, w, s);
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_skeleton_voxels = S;
    if (stats) std::memcpy(stats, st, sizeof(st));
    return CFB_OK;
  });
}

extern "C" int cfb_skeleton_read(void* d_buffer, int64_t z, int64_t y, int64_t x, const double* voxel_size, int64_t num_objects,
                                 int64_t num_voxels, int64_t num_skeleton_voxels, int64_t* num_labels, uint64_t* label_ids,
                                 int64_t* vertex_offsets, int64_t* edge_offsets, float* vertices, uint32_t* edges, float* radii, void* stream) {
  return guarded([&]() -> int {
    const SkGeom g = sk_geom(z, y, x, voxel_size);
    const int64_t K = num_objects, m = num_voxels, S = num_skeleton_voxels;
    if (!num_labels || !vertex_offsets || !edge_offsets || K < 0 || S < K || S > m) throw std::invalid_argument("skeletonize read: bad argument");
    *num_labels = 0;
    vertex_offsets[0] = edge_offsets[0] = 0;
    if (S == 0) return CFB_OK;
    if (!d_buffer || !label_ids || !vertices || !radii || (S > K && !edges)) throw std::invalid_argument("skeletonize read: null argument");
    const SkBuffer b = sk_buffer(d_buffer, K, m);
    cudaStream_t s = (cudaStream_t)stream;
    std::vector<uint32_t> path((size_t)S);
    std::vector<unsigned long long> id((size_t)S), val((size_t)S);
    CFB_CUDA(cudaMemcpyAsync(path.data(), b.path, (size_t)S * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(id.data(), b.ids, (size_t)S * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(val.data(), b.vals, (size_t)S * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> order((size_t)S);
    std::iota(order.begin(), order.end(), 0u);
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t c) { return id[a] != id[c] ? id[a] < id[c] : path[a] < path[c]; });
    int64_t labels = 0, e = 0;
    for (size_t i = 0; i < order.size();) {
      size_t j = i;
      while (j < order.size() && id[order[j]] == id[order[i]]) ++j;
      if (labels >= K) throw std::runtime_error("skeletonize read: more labels than objects");
      std::vector<uint32_t> vox(j - i);
      for (size_t k = i; k < j; ++k) vox[k - i] = path[order[k]];
      for (size_t k = i; k < j; ++k) {
        const uint32_t p = path[order[k]], par = (uint32_t)(val[order[k]] & 0xFFFFFFFFULL);
        const int64_t vi = (int64_t)k;
        const int64_t c[3] = {(int64_t)p / (g.Y * g.X), ((int64_t)p / g.X) % g.Y, (int64_t)p % g.X};
        for (int a = 0; a < 3; ++a) vertices[3 * vi + a] = (float)(((double)c[2 - a] + 0.5) * g.w[2 - a]);
        const uint32_t bits = (uint32_t)(val[order[k]] >> 32);
        std::memcpy(&radii[vi], &bits, 4);
        if (par == p) continue;
        const auto it = std::lower_bound(vox.begin(), vox.end(), par);
        if (it == vox.end() || *it != par) throw std::runtime_error("skeletonize read: a parent is not on the skeleton");
        edges[2 * e] = (uint32_t)(k - i);
        edges[2 * e + 1] = (uint32_t)(it - vox.begin());
        ++e;
      }
      label_ids[labels] = id[order[i]];
      ++labels;
      vertex_offsets[labels] = (int64_t)j;
      edge_offsets[labels] = e;
      i = j;
    }
    if (e != S - K) throw std::runtime_error("skeletonize read: the skeletons are not one tree per object");
    *num_labels = labels;
    return CFB_OK;
  });
}
