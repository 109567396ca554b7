// `mesh` (reference flow/flow.py:2087-2135, flow/mesh.py -> zmesh): marching cubes of every object of a segmentation chunk,
// restated in oracle/mesh_oracle.py (zmesh is not vendored; its meshes are not reproduced).  On the device
// (mesh_kernels.cuh): count the (cube, object) pairs and the (object, cut edge) vertices, so that the caller allocates once;
// emit both streams in order; sort both stably by id; number the objects; give every pair its first face; weld every face
// corner to the rank of its edge key among its object's vertices; place the vertices.  Only the finished meshes come to the
// host.  The simplifier (Garland-Heckbert edge collapse, fully ordered) is host code, like zmesh's: objects are independent
// and are spread over threads by the caller.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iterator>
#include <queue>
#include <stdexcept>
#include <tuple>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

constexpr int kMcThreads = 256;

#include "mesh_kernels.cuh"
#include "raster_scan.cuh"
#include "radix_sort.cuh"

McGrid mc_grid(int64_t z, int64_t y, int64_t x, int32_t close) {
  if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX) throw std::invalid_argument("mesh: bad volume size");
  McGrid g;
  g.Z = z; g.Y = y; g.X = x;
  g.off = close ? -1 : 0;
  const int64_t d = close ? 1 : -1;   // cubes per axis: extent + 1 (closed) or extent - 1 (open)
  g.c[0] = x + d; g.c[1] = y + d; g.c[2] = z + d;
  g.cubes = g.c[0] * g.c[1] * g.c[2];   // 0 when an axis has one voxel and the mesh is open
  g.cells = (z + 2) * (y + 2) * (x + 2);
  return g;
}

int64_t mc_blocks(int64_t items) { return ceil_div64(items, kMcBlock); }

void mc_check(const void* d_labels, int32_t dtype, const void* d_skip, int64_t num_skip, const void* d_workspace) {
  if (!d_labels || !d_workspace) throw std::invalid_argument("mesh: null argument");
  if (dtype != CFB_DTYPE_U32 && dtype != CFB_DTYPE_U64) throw std::invalid_argument("mesh: the ids are uint32 or uint64");
  if (num_skip < 0 || (num_skip > 0 && !d_skip)) throw std::invalid_argument("mesh: bad skip list");
}

// workspace: stats (pairs' triangles, pairs, -, vertices: 4 x 8 B) | block counts and total of the pairs | of the vertices (4 B)
struct McWork {
  unsigned long long* stats;
  uint32_t *pair_blocks, *vert_blocks;
};

McWork mc_work(void* d_workspace, const McGrid& g) {
  McWork w;
  w.stats = static_cast<unsigned long long*>(d_workspace);
  w.pair_blocks = reinterpret_cast<uint32_t*>(w.stats + 4);
  w.vert_blocks = w.pair_blocks + mc_blocks(g.cubes) + 1;
  return w;
}

int64_t mc_workspace_bytes(const McGrid& g) { return 4 * 8 + (mc_blocks(g.cubes) + 1 + mc_blocks(g.cells) + 1) * 4; }

// Buffer of the device weld, for P pairs, V vertices and T triangles (8 B words first):
//   pair ids, codes and their sorted copies (4 P x 8 B) | vertex ids, keys and copies (4 V x 8 B) | object ids (P x 8 B) |
//   pair flags, ranks, first faces (3 P x 4 B) | vertex flags, ranks (2 V x 4 B) | object starts in the pairs, in the vertices,
//   first faces ((P + 1) x 4 B each) | histograms (256 chunks(max(P, V)) x 4 B) | scan sums (chunks + 1 of that x 4 B) |
//   faces (3 T x 4 B) | positions (3 V x 4 B)
struct McBuffer {
  unsigned long long *pid, *pcode, *pid2, *pcode2, *vid, *vkey, *vid2, *vkey2, *object_ids;
  uint32_t *pflag, *prank, *pface, *vflag, *vrank, *obj_pair, *obj_vert, *obj_face, *hist, *sums, *faces;
  float* positions;
  int64_t bytes;
};

McBuffer mc_buffer(void* base, int64_t P, int64_t V, int64_t T) {
  McBuffer b;
  unsigned long long* w = static_cast<unsigned long long*>(base);
  b.pid = w; b.pcode = w + P; b.pid2 = w + 2 * P; b.pcode2 = w + 3 * P;
  w += 4 * P;
  b.vid = w; b.vkey = w + V; b.vid2 = w + 2 * V; b.vkey2 = w + 3 * V;
  w += 4 * V;
  b.object_ids = w;
  w += P;
  uint32_t* u = reinterpret_cast<uint32_t*>(w);
  b.pflag = u; b.prank = u + P; b.pface = u + 2 * P;
  u += 3 * P;
  b.vflag = u; b.vrank = u + V;
  u += 2 * V;
  b.obj_pair = u; b.obj_vert = u + (P + 1); b.obj_face = u + 2 * (P + 1);
  u += 3 * (P + 1);
  const int64_t hist_len = 256 * mc_chunks(std::max(P, V));
  const int64_t scan_max = std::max(hist_len, std::max(P, V));
  b.hist = u;
  u += hist_len;
  b.sums = u;
  u += mc_chunks(scan_max) + 1;
  b.faces = u;
  u += 3 * T;
  b.positions = reinterpret_cast<float*>(u);
  u += 3 * V;
  b.bytes = (int64_t)((char*)u - (char*)base);
  return b;
}

// runs of equal ids of a sorted stream: flag, rank (object of every item), start of every object -> objects
uint32_t mc_objects(const unsigned long long* ids, int64_t n, uint32_t* flag, uint32_t* rank, uint32_t* start, unsigned long long* object_ids,
                    uint32_t* sums, cudaStream_t s) {
  launch(mc_flag_kernel, mc_grid_size(n), kMcThreads, 0, s, ids, n, flag);
  CFB_CUDA(cudaMemcpyAsync(rank, flag, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  const uint32_t objects = mc_scan(rank, n, sums, s);   // rank of a run's first item = its object
  launch(mc_starts_kernel, mc_grid_size(n), kMcThreads, 0, s, ids, n, (const uint32_t*)rank, start, object_ids);
  const uint32_t end = (uint32_t)n;
  CFB_CUDA(cudaMemcpyAsync(start + objects, &end, 4, cudaMemcpyHostToDevice, s));
  CFB_CUDA(cudaStreamSynchronize(s));
  return objects;
}

// the object of every item of a sorted stream: rank[i] = objects started at or before i, minus one
__global__ void __launch_bounds__(kMcThreads) mc_item_object_kernel(const uint32_t* __restrict__ flag, uint32_t* __restrict__ rank, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) rank[i] = rank[i] + flag[i] - 1u;
}

// first face of every object
__global__ void __launch_bounds__(kMcThreads) mc_object_faces_kernel(const uint32_t* __restrict__ obj_pair, const uint32_t* __restrict__ pface,
                                                                      int64_t objects, uint32_t total, uint32_t* __restrict__ obj_face) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o <= objects; o += stride)
    obj_face[o] = o == objects ? total : pface[obj_pair[o]];
}

template <typename T>
void mc_launch_count(const T* seg, const McGrid& g, const unsigned long long* skip, int64_t num_skip, const McWork& w, cudaStream_t s) {
  if (g.cubes) {
    launch(mc_count_kernel<true, T>, mc_grid_size(mc_blocks(g.cubes) * kMcThreads), kMcThreads, 0, s, seg, g, skip, num_skip, g.cubes,
           w.pair_blocks, w.stats);
    launch(mc_count_kernel<false, T>, mc_grid_size(mc_blocks(g.cells) * kMcThreads), kMcThreads, 0, s, seg, g, skip, num_skip, g.cells,
           w.vert_blocks, w.stats + 2);
    launch(cc_scan_blocks_kernel, 1, 1024, 0, s, w.pair_blocks, mc_blocks(g.cubes), w.pair_blocks + mc_blocks(g.cubes));
    launch(cc_scan_blocks_kernel, 1, 1024, 0, s, w.vert_blocks, mc_blocks(g.cells), w.vert_blocks + mc_blocks(g.cells));
  }
}

template <typename T>
void mc_launch_emit(const T* seg, const McGrid& g, const unsigned long long* skip, int64_t num_skip, const McWork& w, const McBuffer& b,
                    cudaStream_t s) {
  launch(mc_emit_kernel<true, T>, mc_grid_size(mc_blocks(g.cubes) * kMcThreads), kMcThreads, 0, s, seg, g, skip, num_skip, g.cubes,
         (const uint32_t*)w.pair_blocks, b.pid, b.pcode);
  launch(mc_emit_kernel<false, T>, mc_grid_size(mc_blocks(g.cells) * kMcThreads), kMcThreads, 0, s, seg, g, skip, num_skip, g.cells,
         (const uint32_t*)w.vert_blocks, b.vid, b.vkey);
}

// ---- the simplifier --------------------------------------------------------------------------------------------------
typedef std::array<double, 10> Quadric;   // a2, ab, ac, ad, b2, bc, bd, c2, cd, d2 of a plane ax + by + cz + d = 0
struct Vec3 { double x, y, z; };

Vec3 sub(const Vec3& a, const Vec3& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
Vec3 cross(const Vec3& a, const Vec3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
double dot(const Vec3& a, const Vec3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

Quadric face_quadric(const Vec3& p0, const Vec3& p1, const Vec3& p2) {
  const Vec3 n = cross(sub(p1, p0), sub(p2, p0));
  const double ln = std::sqrt(n.x * n.x + n.y * n.y + n.z * n.z);
  Quadric q{};
  if (ln == 0.0) return q;
  const double a = n.x / ln, b = n.y / ln, c = n.z / ln;
  const double d = -(a * p0.x + b * p0.y + c * p0.z);
  q = {a * a, a * b, a * c, a * d, b * b, b * c, b * d, c * c, c * d, d * d};
  return q;
}

double quadric_error(const Quadric& q, const Vec3& v) {
  const double x = v.x, y = v.y, z = v.z;
  return q[0] * x * x + 2.0 * q[1] * x * y + 2.0 * q[2] * x * z + 2.0 * q[3] * x + q[4] * y * y + 2.0 * q[5] * y * z +
         2.0 * q[6] * y + q[7] * z * z + 2.0 * q[8] * z + q[9];
}

Quadric add(const Quadric& a, const Quadric& b) {
  Quadric q;
  for (int k = 0; k < 10; ++k) q[k] = a[k] + b[k];
  return q;
}

struct Candidate {
  double cost;
  uint32_t a, b;
  bool operator>(const Candidate& o) const { return std::tie(cost, a, b) > std::tie(o.cost, o.a, o.b); }
};

class Simplifier {
 public:
  Simplifier(int64_t nv, const float* v, int64_t nf, const uint32_t* f) : V_((size_t)nv), Q_((size_t)nv), vf_((size_t)nv),
                                                                             locked_((size_t)nv, 0), F_((size_t)nf), alive_((size_t)nf, 1) {
    for (int64_t i = 0; i < nv; ++i) V_[(size_t)i] = {v[3 * i], v[3 * i + 1], v[3 * i + 2]};
    for (int64_t i = 0; i < nf; ++i) {
      for (int k = 0; k < 3; ++k) {
        if ((int64_t)f[3 * i + k] >= nv) throw std::invalid_argument("mesh simplify: a face index is out of range");
        F_[(size_t)i][k] = f[3 * i + k];
      }
    }
  }

  // -> faces left
  int64_t run(int64_t target, double limit) {
    const size_t nf = F_.size();
    for (size_t i = 0; i < nf; ++i) {
      const auto& f = F_[i];
      const Quadric q = face_quadric(V_[f[0]], V_[f[1]], V_[f[2]]);
      for (int k = 0; k < 3; ++k) {
        Q_[f[k]] = add(Q_[f[k]], q);
        vf_[f[k]].push_back((uint32_t)i);
      }
    }
    std::vector<uint64_t> edges;   // (min << 32 | max), one per face side
    edges.reserve(3 * nf);
    for (const auto& f : F_)
      for (int k = 0; k < 3; ++k) {
        const uint32_t a = f[k], b = f[(k + 1) % 3];
        edges.push_back((uint64_t)std::min(a, b) << 32 | std::max(a, b));
      }
    std::sort(edges.begin(), edges.end());
    for (size_t i = 0; i < edges.size();) {   // an edge of one face only: an open border, its ends stay
      size_t j = i;
      while (j < edges.size() && edges[j] == edges[i]) ++j;
      if (j - i == 1) locked_[edges[i] >> 32] = locked_[edges[i] & 0xffffffffu] = 1;
      i = j;
    }
    edges.erase(std::unique(edges.begin(), edges.end()), edges.end());
    std::vector<Candidate> init;
    for (const uint64_t e : edges) {
      Candidate c;
      Vec3 p;
      if (candidate((uint32_t)(e >> 32), (uint32_t)e, c, p)) init.push_back(c);
    }
    std::priority_queue<Candidate, std::vector<Candidate>, std::greater<Candidate>> heap(std::greater<Candidate>(), std::move(init));
    int64_t left = (int64_t)nf;
    while (left > target && !heap.empty()) {
      const Candidate top = heap.top();
      heap.pop();
      if (top.cost > limit) break;
      const uint32_t a = top.a, b = top.b;
      std::vector<uint32_t> shared;
      for (const uint32_t fi : vf_[a])
        if (std::find(vf_[b].begin(), vf_[b].end(), fi) != vf_[b].end()) shared.push_back(fi);
      if (shared.empty()) continue;   // no longer an edge
      Candidate c;
      Vec3 p;
      if (!candidate(a, b, c, p)) continue;
      if (c.cost != top.cost) { heap.push(c); continue; }   // stale: again with the current cost
      if (!collapse_ok(a, b, p, shared)) continue;
      for (const uint32_t fi : shared) {
        alive_[fi] = 0;
        for (int k = 0; k < 3; ++k) erase(vf_[F_[fi][k]], fi);
        --left;
      }
      for (const uint32_t fi : vf_[b]) {
        for (int k = 0; k < 3; ++k)
          if (F_[fi][k] == b) F_[fi][k] = a;
        vf_[a].push_back(fi);
      }
      vf_[b].clear();
      V_[a] = {(double)(float)p.x, (double)(float)p.y, (double)(float)p.z};
      Q_[a] = add(Q_[a], Q_[b]);
      locked_[a] |= locked_[b];   // a border vertex stays where it is
      // every edge whose cost or whose test can have changed: those of a and of its neighbours (a refused collapse comes back)
      std::vector<uint32_t> nbrs, around;
      ring(a, nbrs);
      nbrs.insert(nbrs.begin(), a);
      for (const uint32_t u : nbrs) {
        ring(u, around);
        for (const uint32_t w : around) {
          Candidate c2;
          Vec3 p2;
          if (candidate(std::min(u, w), std::max(u, w), c2, p2)) heap.push(c2);
        }
      }
    }
    return left;
  }

  // kept faces in their order, vertices renumbered in order of first use
  void write(float* out_v, uint32_t* out_f, int64_t* out_nv) const {
    std::vector<uint32_t> remap(V_.size(), UINT32_MAX);
    uint32_t nv = 0;
    int64_t j = 0;
    for (size_t i = 0; i < F_.size(); ++i) {
      if (!alive_[i]) continue;
      for (int k = 0; k < 3; ++k) {
        const uint32_t v = F_[i][k];
        if (remap[v] == UINT32_MAX) {
          out_v[3 * nv] = (float)V_[v].x; out_v[3 * nv + 1] = (float)V_[v].y; out_v[3 * nv + 2] = (float)V_[v].z;
          remap[v] = nv++;
        }
        out_f[j++] = remap[v];
      }
    }
    *out_nv = nv;
  }

 private:
  static void erase(std::vector<uint32_t>& v, uint32_t x) { v.erase(std::remove(v.begin(), v.end(), x), v.end()); }

  bool candidate(uint32_t a, uint32_t b, Candidate& c, Vec3& p) const {
    if (locked_[a] && locked_[b]) return false;
    const Quadric q = add(Q_[a], Q_[b]);
    if (locked_[a]) {
      p = V_[a];
    } else if (locked_[b]) {
      p = V_[b];
    } else {
      const Vec3 mid = {(V_[a].x + V_[b].x) * 0.5, (V_[a].y + V_[b].y) * 0.5, (V_[a].z + V_[b].z) * 0.5};
      const Vec3 opts[3] = {V_[a], V_[b], mid};
      double best = 0.0;
      for (int k = 0; k < 3; ++k) {
        const double e = quadric_error(q, opts[k]);
        if (k == 0 || e < best) { best = e; p = opts[k]; }
      }
    }
    c = {quadric_error(q, p), a, b};
    return true;
  }

  void ring(uint32_t v, std::vector<uint32_t>& out) const {
    out.clear();
    for (const uint32_t fi : vf_[v])
      for (int k = 0; k < 3; ++k)
        if (F_[fi][k] != v) out.push_back(F_[fi][k]);
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
  }

  bool collapse_ok(uint32_t a, uint32_t b, const Vec3& p, const std::vector<uint32_t>& shared) const {
    std::vector<uint32_t> na, nb, common, opposite;
    ring(a, na);
    ring(b, nb);
    std::set_intersection(na.begin(), na.end(), nb.begin(), nb.end(), std::back_inserter(common));
    erase_pair(common, a, b);
    for (const uint32_t fi : shared)
      for (int k = 0; k < 3; ++k)
        if (F_[fi][k] != a && F_[fi][k] != b) opposite.push_back(F_[fi][k]);
    std::sort(opposite.begin(), opposite.end());
    opposite.erase(std::unique(opposite.begin(), opposite.end()), opposite.end());
    if (common != opposite) return false;   // link condition
    auto is_shared = [&](uint32_t fi) { return std::find(shared.begin(), shared.end(), fi) != shared.end(); };
    std::vector<std::array<uint32_t, 3>> existing;   // sorted vertex sets of a's faces that stay
    for (const uint32_t fi : vf_[a])
      if (!is_shared(fi)) existing.push_back(sorted(F_[fi]));
    for (int side = 0; side < 2; ++side) {
      for (const uint32_t fi : vf_[side ? b : a]) {
        if (is_shared(fi)) continue;
        const auto& f = F_[fi];
        if (side) {
          std::array<uint32_t, 3> g = f;
          for (auto& i : g)
            if (i == b) i = a;
          if (std::find(existing.begin(), existing.end(), sorted(g)) != existing.end()) return false;
        }
        Vec3 o[3], n[3];
        for (int k = 0; k < 3; ++k) {
          o[k] = V_[f[k]];
          n[k] = (f[k] == a || f[k] == b) ? p : V_[f[k]];
        }
        const Vec3 n0 = cross(sub(o[1], o[0]), sub(o[2], o[0]));
        const Vec3 n1 = cross(sub(n[1], n[0]), sub(n[2], n[0]));
        if (dot(n1, n1) == 0.0 || dot(n0, n1) <= 0.0) return false;
      }
    }
    return true;
  }

  static void erase_pair(std::vector<uint32_t>& v, uint32_t a, uint32_t b) {
    v.erase(std::remove_if(v.begin(), v.end(), [&](uint32_t x) { return x == a || x == b; }), v.end());
  }

  static std::array<uint32_t, 3> sorted(std::array<uint32_t, 3> f) {
    std::sort(f.begin(), f.end());
    return f;
  }

  std::vector<Vec3> V_;
  std::vector<Quadric> Q_;
  std::vector<std::vector<uint32_t>> vf_;
  std::vector<uint8_t> locked_;
  std::vector<std::array<uint32_t, 3>> F_;
  std::vector<uint8_t> alive_;
};

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_mesh_workspace(int64_t z, int64_t y, int64_t x, int32_t close, int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    if (!workspace_bytes) throw std::invalid_argument("mesh: null output");
    *workspace_bytes = mc_workspace_bytes(mc_grid(z, y, x, close));
    return CFB_OK;
  });
}

extern "C" int cfb_mesh_count_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const uint64_t* d_skip_ids,
                                     int64_t num_skip, int32_t close, void* d_workspace, int64_t* num_pairs, int64_t* num_triangles,
                                     int64_t* num_vertices, void* stream) {
  return guarded([&]() -> int {
    mc_check(d_labels, dtype, d_skip_ids, num_skip, d_workspace);
    if (!num_pairs || !num_triangles || !num_vertices) throw std::invalid_argument("mesh: null output");
    const McGrid g = mc_grid(z, y, x, close);
    cudaStream_t s = (cudaStream_t)stream;
    const McWork w = mc_work(d_workspace, g);
    CFB_CUDA(cudaMemsetAsync(w.stats, 0, 4 * 8, s));
    const unsigned long long* skip = (const unsigned long long*)d_skip_ids;
    if (dtype == CFB_DTYPE_U32) mc_launch_count((const uint32_t*)d_labels, g, skip, num_skip, w, s);
    else mc_launch_count((const uint64_t*)d_labels, g, skip, num_skip, w, s);
    unsigned long long h[4];
    CFB_CUDA(cudaMemcpyAsync(h, w.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (h[0] >= UINT32_MAX || h[3] >= UINT32_MAX || 256 * mc_chunks((int64_t)std::max(h[1], h[3])) >= (int64_t)UINT32_MAX)
      throw std::invalid_argument("mesh: 2^32 or more triangles or vertices in one chunk");
    *num_triangles = (int64_t)h[0];
    *num_pairs = (int64_t)h[1];
    *num_vertices = (int64_t)h[3];
    return CFB_OK;
  });
}

extern "C" int cfb_mesh_buffer_bytes(int64_t num_pairs, int64_t num_triangles, int64_t num_vertices, int64_t* buffer_bytes) {
  return guarded([&]() -> int {
    if (num_pairs < 0 || num_triangles < 0 || num_vertices < 0 || !buffer_bytes) throw std::invalid_argument("mesh: bad counts");
    *buffer_bytes = mc_buffer(nullptr, num_pairs, num_vertices, num_triangles).bytes;
    return CFB_OK;
  });
}

extern "C" int cfb_mesh_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const uint64_t* d_skip_ids,
                               int64_t num_skip, int32_t close, const double* voxel_size, void* d_workspace, int64_t num_pairs,
                               int64_t num_triangles, int64_t num_vertices, void* d_buffer, int64_t buffer_bytes, int64_t* num_objects,
                               void* stream) {
  return guarded([&]() -> int {
    mc_check(d_labels, dtype, d_skip_ids, num_skip, d_workspace);
    if (!voxel_size || !num_objects || !d_buffer) throw std::invalid_argument("mesh: null argument");
    const McGrid g = mc_grid(z, y, x, close);
    const McBuffer b = mc_buffer(d_buffer, num_pairs, num_vertices, num_triangles);
    if (num_pairs < 0 || buffer_bytes < b.bytes) throw std::invalid_argument("mesh: the buffer is smaller than cfb_mesh_buffer_bytes");
    cudaStream_t s = (cudaStream_t)stream;
    const McWork w = mc_work(d_workspace, g);
    unsigned long long h[4];
    CFB_CUDA(cudaMemcpyAsync(h, w.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if ((int64_t)h[1] != num_pairs || (int64_t)h[0] != num_triangles || (int64_t)h[3] != num_vertices)
      throw std::invalid_argument("mesh: the counts are not those of cfb_mesh_count_device for this volume");
    *num_objects = 0;
    if (num_pairs == 0) return CFB_OK;
    const unsigned long long* skip = (const unsigned long long*)d_skip_ids;
    if (dtype == CFB_DTYPE_U32) mc_launch_emit((const uint32_t*)d_labels, g, skip, num_skip, w, b, s);
    else mc_launch_emit((const uint64_t*)d_labels, g, skip, num_skip, w, b, s);
    const int bits = dtype == CFB_DTYPE_U32 ? 32 : 64;
    mc_sort(b.pid, b.pcode, b.pid2, b.pcode2, num_pairs, bits, b.hist, b.sums, s);
    mc_sort(b.vid, b.vkey, b.vid2, b.vkey2, num_vertices, bits, b.hist, b.sums, s);
    const uint32_t objects = mc_objects(b.pid, num_pairs, b.pflag, b.prank, b.obj_pair, b.object_ids, b.sums, s);
    const uint32_t vobjects = mc_objects(b.vid, num_vertices, b.vflag, b.vrank, b.obj_vert, nullptr, b.sums, s);
    if (objects != vobjects) throw std::runtime_error("mesh: the pairs and the vertices name different objects");
    launch(mc_item_object_kernel, mc_grid_size(num_pairs), kMcThreads, 0, s, (const uint32_t*)b.pflag, b.prank, num_pairs);
    launch(mc_tri_count_kernel, mc_grid_size(num_pairs), kMcThreads, 0, s, (const unsigned long long*)b.pcode, num_pairs, b.pface);
    const uint32_t faces = mc_scan(b.pface, num_pairs, b.sums, s);
    if ((int64_t)faces != num_triangles) throw std::runtime_error("mesh: the emitted pairs do not hold the counted triangles");
    launch(mc_object_faces_kernel, mc_grid_size(objects + 1), kMcThreads, 0, s, (const uint32_t*)b.obj_pair, (const uint32_t*)b.pface,
           (int64_t)objects, faces, b.obj_face);
    launch(mc_faces_kernel, mc_grid_size(num_pairs), kMcThreads, 0, s, g, (const unsigned long long*)b.pcode, num_pairs,
           (const uint32_t*)b.pface, (const uint32_t*)b.prank, (const uint32_t*)b.obj_vert, (const unsigned long long*)b.vkey, b.faces);
    launch(mc_positions_kernel, mc_grid_size(num_vertices), kMcThreads, 0, s, g, (const unsigned long long*)b.vkey, num_vertices,
           voxel_size[2], voxel_size[1], voxel_size[0], b.positions);
    *num_objects = objects;
    return CFB_OK;
  });
}

extern "C" int cfb_mesh_read(void* d_buffer, int64_t num_pairs, int64_t num_triangles, int64_t num_vertices, int64_t num_objects,
                             uint64_t* object_ids, int64_t* face_offsets, int64_t* vertex_offsets, uint32_t* faces, float* vertices,
                             void* stream) {
  return guarded([&]() -> int {
    if (!d_buffer || num_objects < 0 || num_objects > num_pairs) throw std::invalid_argument("mesh read: bad argument");
    if (num_objects == 0) return CFB_OK;
    if (!object_ids || !face_offsets || !vertex_offsets || !faces || !vertices) throw std::invalid_argument("mesh read: null output");
    const McBuffer b = mc_buffer(d_buffer, num_pairs, num_vertices, num_triangles);
    cudaStream_t s = (cudaStream_t)stream;
    std::vector<uint32_t> fo((size_t)num_objects + 1), vo((size_t)num_objects + 1);
    CFB_CUDA(cudaMemcpyAsync(object_ids, b.object_ids, (size_t)num_objects * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(fo.data(), b.obj_face, fo.size() * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(vo.data(), b.obj_vert, vo.size() * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(faces, b.faces, (size_t)num_triangles * 12, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(vertices, b.positions, (size_t)num_vertices * 12, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    for (int64_t o = 0; o <= num_objects; ++o) {
      face_offsets[o] = fo[(size_t)o];
      vertex_offsets[o] = vo[(size_t)o];
    }
    if (face_offsets[num_objects] != num_triangles || vertex_offsets[num_objects] != num_vertices)
      throw std::invalid_argument("mesh read: the counts are not those of the buffer");
    return CFB_OK;
  });
}

extern "C" int cfb_mesh_simplify_host(int64_t num_vertices, const float* vertices, int64_t num_faces, const uint32_t* faces,
                                      int64_t simplification_factor, double max_simplification_error, int64_t* out_num_vertices,
                                      float* out_vertices, int64_t* out_num_faces, uint32_t* out_faces) {
  return guarded([&]() -> int {
    if (num_vertices < 0 || num_faces < 0 || num_vertices >= (int64_t)UINT32_MAX || !out_num_vertices || !out_num_faces)
      throw std::invalid_argument("mesh simplify: bad argument");
    if ((num_vertices && (!vertices || !out_vertices)) || (num_faces && (!faces || !out_faces)))
      throw std::invalid_argument("mesh simplify: null array");
    if (simplification_factor <= 1) {   // unchanged
      if (num_vertices) std::memcpy(out_vertices, vertices, (size_t)num_vertices * 3 * sizeof(float));
      if (num_faces) std::memcpy(out_faces, faces, (size_t)num_faces * 3 * sizeof(uint32_t));
      *out_num_vertices = num_vertices;
      *out_num_faces = num_faces;
      return CFB_OK;
    }
    Simplifier s(num_vertices, vertices, num_faces, faces);
    const int64_t target = ceil_div64(num_faces, simplification_factor);
    *out_num_faces = s.run(target, max_simplification_error * max_simplification_error);
    s.write(out_vertices, out_faces, out_num_vertices);
    return CFB_OK;
  });
}
