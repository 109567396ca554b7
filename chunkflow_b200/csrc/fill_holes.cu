// `fill-segmentation-holes` (reference chunkflow/plugins/fill_segmentation_holes.py -> fill_voids.fill), rules restated in
// oracle/fill_holes_oracle.py (fill_voids is not vendored).  Every connectivity is 6 (face neighbours); "outside" is the space
// beyond the chunk's six faces, which every face voxel reaches.
//   components  union-find over the 6 neighbours (union_find.cuh): of the background alone (binary), or of every value, 0
//               included (per-object modes); flattened, numbered 0 .. C - 1 in raster order of their first voxel by an
//               exclusive scan of the root flags (radix_sort.cuh: mc_scan); one pass over the six faces flags the components
//               that reach outside.  A background component without the flag is a hole.
//   graph       (per-object modes) the distinct pairs of touching components in an open-addressing table (hash_table.cuh),
//               runs of equal pairs in a warp's 32 consecutive voxels inserted once; CFB_ERR_CAPACITY when it is too full.
//   enclose     (per-object modes, on the host) a virtual root joined to the flagged components, an iterative Hopcroft-Tarjan
//               DFS from it, and each component's innermost and outermost non-zero encloser propagated down the DFS tree: a
//               component's enclosers are the cut vertices between it and the root, i.e. its DFS ancestors p (not the root)
//               whose child c on the path has low[c] >= disc[p]; deeper is inner.  -> a target component per component.
//   apply       one pass writes the output in the input's dtype and counts the voxels the rule assigns.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

constexpr int kFhThreads = 256;
constexpr int kMcThreads = kFhThreads;   // radix_sort.cuh
constexpr uint32_t kFhNone = 0xFFFFFFFFu;

#include "union_find.cuh"
#include "raster_scan.cuh"
#include "radix_sort.cuh"
#include "state_table.cuh"   // ev_lane / ev_shfl_up / ev_warp_sum and hash_table.cuh

int fh_grid(int64_t work) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(work, kFhThreads), 132 * 16)); }

// a voxel takes part in the components: every voxel in the per-object modes, the background (value 0) in binary mode
template <typename T, bool kBinary>
__device__ __forceinline__ bool fh_member(const T* __restrict__ seg, int64_t i) { return !kBinary || !seg[i]; }

__global__ void __launch_bounds__(kFhThreads) fh_init_kernel(uint32_t* __restrict__ P, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) P[i] = (uint32_t)i;
}

// P[i] = root(i); flag[i] = 1 at the root of a member component (the scan turns the flags into component numbers)
template <typename T, bool kBinary>
__global__ void __launch_bounds__(kFhThreads) fh_flatten_kernel(const T* __restrict__ seg, uint32_t* __restrict__ P, uint32_t* __restrict__ flag,
                                                               int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const bool m = fh_member<T, kBinary>(seg, i);
    uint32_t r = (uint32_t)i;
    if (m) {
      r = uf_find(P, (uint32_t)i);
      P[i] = r;   // (roots keep P[r] == r; concurrent readers only ever see an ancestor)
    }
    flag[i] = m && r == (uint32_t)i;
  }
}

// P[i] = the component of a member voxel; at the root, root[c] = its voxel and flags[c] = 2 when its value is not 0
template <typename T, bool kBinary>
__global__ void __launch_bounds__(kFhThreads) fh_label_kernel(const T* __restrict__ seg, uint32_t* __restrict__ P, const uint32_t* __restrict__ rank,
                                                             uint32_t* __restrict__ root, uint8_t* __restrict__ flags, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (!fh_member<T, kBinary>(seg, i)) continue;
    const uint32_t r = P[i], c = rank[r];
    if (r == (uint32_t)i) {
      root[c] = r;
      flags[c] = seg[i] ? 2 : 0;
    }
    P[i] = c;
  }
}

// flags[c] |= 1 for the member components with a voxel on one of the six faces (z = 0, Z - 1, then y, then x; the edges are
// visited more than once, and concurrent writers of a component store the same byte)
template <typename T, bool kBinary>
__global__ void __launch_bounds__(kFhThreads) fh_face_kernel(const T* __restrict__ seg, const uint32_t* __restrict__ comp, Int3 sz,
                                                            uint8_t* __restrict__ flags) {
  const int64_t Z = sz.z, Y = sz.y, X = sz.x;
  const int64_t a = 2 * Y * X, b = a + 2 * Z * X, total = b + 2 * Z * Y;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
    int64_t z, y, x;
    if (k < a) { z = (k / (Y * X)) ? Z - 1 : 0; y = (k / X) % Y; x = k % X; }
    else if (k < b) { const int64_t q = k - a; y = (q / (Z * X)) ? Y - 1 : 0; z = (q / X) % Z; x = q % X; }
    else { const int64_t q = k - b; x = (q / (Z * Y)) ? X - 1 : 0; z = (q / Y) % Z; y = q % Y; }
    const int64_t i = (z * Y + y) * X + x;
    if (!fh_member<T, kBinary>(seg, i)) continue;
    const uint32_t c = comp[i];
    if (!(flags[c] & 1)) flags[c] |= 1;
  }
}

// the distinct pairs of touching components, key (smaller << 32 | larger), never 0: the two differ.  A lane inserts the pair
// of a direction unless the lane before it holds the same one.  info[0] = pairs, info[1] = overflow.
__global__ void __launch_bounds__(kFhThreads) fh_graph_kernel(const uint32_t* __restrict__ comp, Int3 sz, unsigned long long* __restrict__ keys,
                                                             unsigned long long mask, uint32_t* __restrict__ info) {
  const int64_t n = (int64_t)sz.z * sz.y * sz.x, step[3] = {(int64_t)sz.y * sz.x, (int64_t)sz.x, 1};
  const int lane = ev_lane();
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / EV_WARP;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = warp * EV_WARP; base < n; base += stride) {   // warp-uniform: every lane reaches the shuffles
    const int64_t i = base + lane;
    const bool valid = i < n;
    const uint32_t c = valid ? comp[i] : 0u;
    const int coord[3] = {valid ? (int)(i / step[0]) : 0, valid ? (int)((i / sz.x) % sz.y) : 0, valid ? (int)(i % sz.x) : 0};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const uint32_t d = valid && coord[a] > 0 ? comp[i - step[a]] : c;
      const unsigned long long key = c == d ? 0ULL : ((unsigned long long)min(c, d) << 32) | max(c, d);
      const unsigned long long prev = ev_shfl_up(key);
      if (!key || (lane > 0 && prev == key)) continue;
      unsigned long long h = rg_hash(key) & mask;
      bool done = false;
      for (int probe = 0; probe < kRgMaxProbe; ++probe, h = (h + 1) & mask) {
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(keys + h);   // other threads insert concurrently
        if (cur != key) {
          if (cur != 0ULL) continue;
          cur = atomicCAS(&keys[h], 0ULL, key);
          if (cur == 0ULL) atomicAdd(&info[0], 1u);
          else if (cur != key) continue;
        }
        done = true;
        break;
      }
      if (!done) info[1] = 1u;   // table too full: the host retries with a larger one
    }
  }
}

__global__ void __launch_bounds__(kFhThreads) fh_gather_kernel(const unsigned long long* __restrict__ keys, int64_t slots,
                                                              unsigned long long* __restrict__ okeys, uint32_t* __restrict__ cursor) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k) okeys[atomicAdd(cursor, 1u)] = k;
  }
}

__device__ __forceinline__ void fh_count(unsigned long long mine, unsigned long long* count) {
  mine = ev_warp_sum(mine);
  if (ev_lane() == 0 && mine) atomicAdd(count, mine);
}

// binary: 1 for the foreground and the holes (background components that do not reach outside), 0 elsewhere
template <typename T>
__global__ void __launch_bounds__(kFhThreads) fh_apply_binary_kernel(const T* __restrict__ seg, const uint32_t* __restrict__ comp,
                                                                    const uint8_t* __restrict__ flags, T* __restrict__ out, int64_t n,
                                                                    unsigned long long* __restrict__ count) {
  unsigned long long mine = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool one = !!seg[i];
    if (!one) {
      one = !(flags[comp[i]] & 1);
      mine += one;
    }
    out[i] = one ? (T)1 : (T)0;
  }
  fh_count(mine, count);
}

// per object: the value of the target component, or the voxel's own where the map leaves it (kFhNone)
template <typename T>
__global__ void __launch_bounds__(kFhThreads) fh_apply_kernel(const T* __restrict__ seg, const uint32_t* __restrict__ comp,
                                                             const uint32_t* __restrict__ map, const uint32_t* __restrict__ root,
                                                             T* __restrict__ out, int64_t n, unsigned long long* __restrict__ count) {
  unsigned long long mine = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t t = map[comp[i]];
    out[i] = t == kFhNone ? seg[i] : seg[root[t]];
    mine += t != kFhNone;
  }
  fh_count(mine, count);
}

// workspace (8-byte words first): info (8 x 8 B: mode + 1, components, the apply's count, "enclosed") | components (n) |
// root flags, then ranks, then the map (n) | root voxels (n) | scan sums | flags (n x 1 B)
struct FhWork {
  unsigned long long* info;
  uint32_t *comp, *rank, *root, *sums;
  uint8_t* flags;
  int64_t bytes;
};

FhWork fh_work(void* base, int64_t n) {
  FhWork w;
  w.info = static_cast<unsigned long long*>(base);
  w.comp = reinterpret_cast<uint32_t*>(w.info + 8);
  w.rank = w.comp + n;
  w.root = w.rank + n;
  w.sums = w.root + n;
  w.flags = reinterpret_cast<uint8_t*>(w.sums + mc_chunks(n) + 1);
  w.bytes = (int64_t)((char*)(w.flags + n) - (char*)base);
  return w;
}

// pair table: keys | compact keys (slots x 8 B) | info (pairs, overflow, read cursor, spare: 4 x 4 B)
struct FhTable {
  unsigned long long *keys, *okeys;
  uint32_t* info;
  int64_t slots, bytes;
};

FhTable fh_table(void* base, int64_t slots) {
  FhTable t;
  t.slots = slots;
  t.keys = static_cast<unsigned long long*>(base);
  t.okeys = t.keys + slots;
  t.info = reinterpret_cast<uint32_t*>(t.okeys + slots);
  t.bytes = slots * 16 + 16;
  return t;
}

Int3 fh_size(int64_t z, int64_t y, int64_t x) {
  if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX)
    throw std::invalid_argument("fill holes: every axis of the chunk has 1 to 2^31 - 1 voxels");
  if (z * y > ((int64_t)1 << 62) / x || z * y * x >= ((int64_t)1 << 32))
    throw std::invalid_argument("fill holes: the chunk must have fewer than 2^32 voxels");
  return Int3{(int)z, (int)y, (int)x};
}

int64_t fh_voxels(const Int3& s) { return (int64_t)s.z * s.y * s.x; }

void fh_check_slots(int64_t table_slots) {
  if (table_slots < 2 || (table_slots & (table_slots - 1)) || table_slots >= ((int64_t)1 << 31))
    throw std::invalid_argument("fill holes: table_slots must be a power of two below 2^31 (at most 2^30 touching component pairs)");
}

void fh_check_mode(int32_t dtype, int32_t mode) {
  if (mode != CFB_FILL_BINARY && mode != CFB_FILL_KEEP_ENCLOSED && mode != CFB_FILL_REMOVE_ENCLOSED)
    throw std::invalid_argument("fill holes: the mode is binary, keep-enclosed or remove-enclosed");
  if (mode == CFB_FILL_BINARY) {
    if (dtype != CFB_DTYPE_U8 && dtype != CFB_DTYPE_F32 && dtype != CFB_DTYPE_U32 && dtype != CFB_DTYPE_U64)
      throw std::invalid_argument("fill holes: binary mode takes bool, uint8, int32, uint32, int64, uint64 or float32 voxels");
  } else if (dtype != CFB_DTYPE_U32 && dtype != CFB_DTYPE_U64) {
    throw std::invalid_argument("fill holes: the per-object modes take uint32, int32, uint64 or int64 ids");
  }
}

template <typename T, bool kBinary>
uint32_t fh_components(const T* seg, const Int3& sz, const FhWork& w, cudaStream_t s) {
  const int64_t n = fh_voxels(sz);
  launch(fh_init_kernel, fh_grid(n), kFhThreads, 0, s, w.comp, n);
  launch(cc_merge_kernel<T, kBinary ? kJoinZero : kJoinAll>, fh_grid(n), kFhThreads, 0, s, seg, w.comp, sz, 3);
  launch(fh_flatten_kernel<T, kBinary>, fh_grid(n), kFhThreads, 0, s, seg, w.comp, w.rank, n);
  const uint32_t C = mc_scan(w.rank, n, w.sums, s);
  launch(fh_label_kernel<T, kBinary>, fh_grid(n), kFhThreads, 0, s, seg, w.comp, (const uint32_t*)w.rank, w.root, w.flags, n);
  const int64_t faces = 2 * ((int64_t)sz.y * sz.x + (int64_t)sz.z * sz.x + (int64_t)sz.z * sz.y);
  launch(fh_face_kernel<T, kBinary>, fh_grid(faces), kFhThreads, 0, s, seg, (const uint32_t*)w.comp, sz, w.flags);
  return C;
}

template <typename T>
uint32_t fh_components_mode(const void* seg, int32_t mode, const Int3& sz, const FhWork& w, cudaStream_t s) {
  if (mode == CFB_FILL_BINARY) return fh_components<T, true>((const T*)seg, sz, w, s);
  return fh_components<T, false>((const T*)seg, sz, w, s);
}

template <typename T>
void fh_apply(const void* seg, void* out, int32_t mode, int64_t n, const FhWork& w, cudaStream_t s) {
  if (mode == CFB_FILL_BINARY)
    launch(fh_apply_binary_kernel<T>, fh_grid(n), kFhThreads, 0, s, (const T*)seg, (const uint32_t*)w.comp, (const uint8_t*)w.flags, (T*)out, n,
           w.info + 2);
  else
    launch(fh_apply_kernel<T>, fh_grid(n), kFhThreads, 0, s, (const T*)seg, (const uint32_t*)w.comp, (const uint32_t*)w.rank,
           (const uint32_t*)w.root, (T*)out, n, w.info + 2);
}

// info[0 .. 3] of the workspace, checked against what the caller says it holds
void fh_read_info(const FhWork& w, unsigned long long h[4], cudaStream_t s) {
  CFB_CUDA(cudaMemcpyAsync(h, w.info, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  CFB_CUDA(cudaStreamSynchronize(s));
  if (h[0] < 1 || h[0] > 3) throw std::invalid_argument("fill holes: the workspace holds no components (call cfb_fill_holes_components_device)");
}

// The enclosure on the host: the innermost (keep-enclosed, on value-0 components) or outermost (remove-enclosed) non-zero
// encloser of every component, or kFhNone.  Node C is the virtual root (outside).
void fh_enclose_host(int64_t C, const uint8_t* flags, const unsigned long long* pairs, int64_t E, int32_t mode, uint32_t* map) {
  const uint32_t R = (uint32_t)C, V = (uint32_t)(C + 1);
  std::vector<int64_t> off((size_t)V + 1, 0);
  for (int64_t e = 0; e < E; ++e) {
    const uint32_t a = (uint32_t)(pairs[e] >> 32), b = (uint32_t)(pairs[e] & 0xFFFFFFFFULL);
    if (a >= R || b >= R || a == b) throw std::runtime_error("fill holes: a pair names a component that does not exist");
    ++off[a + 1]; ++off[b + 1];
  }
  for (int64_t c = 0; c < C; ++c)
    if (flags[c] & 1) { ++off[c + 1]; ++off[(size_t)R + 1]; }
  for (uint32_t v = 0; v < V; ++v) off[v + 1] += off[v];
  std::vector<uint32_t> adj((size_t)off[V]);
  {
    std::vector<int64_t> at(off.begin(), off.end() - 1);
    for (int64_t e = 0; e < E; ++e) {
      const uint32_t a = (uint32_t)(pairs[e] >> 32), b = (uint32_t)(pairs[e] & 0xFFFFFFFFULL);
      adj[(size_t)at[a]++] = b;
      adj[(size_t)at[b]++] = a;
    }
    for (int64_t c = 0; c < C; ++c)
      if (flags[c] & 1) { adj[(size_t)at[c]++] = R; adj[(size_t)at[R]++] = (uint32_t)c; }
  }
  // iterative DFS from the root: discovery times, low points, tree parents, preorder.  The parent edge is not skipped: it can
  // only lower low[c] to disc[p], which keeps low[c] >= disc[p].
  std::vector<uint32_t> disc((size_t)V, kFhNone), low((size_t)V), parent((size_t)V, kFhNone), order, stack;
  std::vector<int64_t> it(off.begin(), off.end() - 1);
  order.reserve((size_t)V);
  uint32_t t = 0;
  disc[R] = low[R] = t++;
  order.push_back(R);
  stack.push_back(R);
  while (!stack.empty()) {
    const uint32_t v = stack.back();
    if (it[v] < off[(size_t)v + 1]) {
      const uint32_t u = adj[(size_t)it[v]++];
      if (disc[u] == kFhNone) {
        disc[u] = low[u] = t++;
        parent[u] = v;
        order.push_back(u);
        stack.push_back(u);
      } else {
        low[v] = std::min(low[v], disc[u]);
      }
    } else {
      stack.pop_back();
      if (parent[v] != kFhNone) low[parent[v]] = std::min(low[parent[v]], low[v]);
    }
  }
  if ((int64_t)order.size() != (int64_t)V) throw std::runtime_error("fill holes: the component graph is not connected");
  // top down: the enclosers of v are those of its parent p, and p itself when p separates v from the root
  std::vector<uint32_t> inner((size_t)V, kFhNone), outer((size_t)V, kFhNone);
  for (size_t k = 1; k < order.size(); ++k) {
    const uint32_t v = order[k], p = parent[v];
    const bool sep = p != R && low[v] >= disc[p] && (flags[p] & 2);
    inner[v] = sep ? p : inner[p];
    outer[v] = outer[p] != kFhNone ? outer[p] : sep ? p : kFhNone;
  }
  for (int64_t c = 0; c < C; ++c)
    map[c] = mode == CFB_FILL_KEEP_ENCLOSED ? ((flags[c] & 2) ? kFhNone : inner[(size_t)c]) : outer[(size_t)c];
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_fill_holes_workspace(int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    if (!workspace_bytes) throw std::invalid_argument("fill holes: null output");
    *workspace_bytes = fh_work(nullptr, fh_voxels(fh_size(z, y, x))).bytes;
    return CFB_OK;
  });
}

extern "C" int cfb_fill_holes_table_workspace(int64_t table_slots, int64_t* table_bytes) {
  return guarded([&]() -> int {
    if (!table_bytes) throw std::invalid_argument("fill holes: null output");
    fh_check_slots(table_slots);
    *table_bytes = fh_table(nullptr, table_slots).bytes;
    return CFB_OK;
  });
}

extern "C" int cfb_fill_holes_components_device(const void* d_in, int32_t dtype, int64_t z, int64_t y, int64_t x, int32_t mode,
                                                void* d_workspace, int64_t* num_components, void* stream) {
  return guarded([&]() -> int {
    fh_check_mode(dtype, mode);
    if (!d_in || !d_workspace || !num_components) throw std::invalid_argument("fill holes: null argument");
    const Int3 sz = fh_size(z, y, x);
    const FhWork w = fh_work(d_workspace, fh_voxels(sz));
    cudaStream_t s = (cudaStream_t)stream;
    CFB_CUDA(cudaMemsetAsync(w.info, 0, 8 * 8, s));
    CFB_CUDA(cudaMemsetAsync(w.flags, 0, (size_t)fh_voxels(sz), s));
    uint32_t C;
    if (dtype == CFB_DTYPE_U8) C = fh_components_mode<uint8_t>(d_in, mode, sz, w, s);
    else if (dtype == CFB_DTYPE_F32) C = fh_components_mode<float>(d_in, mode, sz, w, s);
    else if (dtype == CFB_DTYPE_U32) C = fh_components_mode<uint32_t>(d_in, mode, sz, w, s);
    else C = fh_components_mode<unsigned long long>(d_in, mode, sz, w, s);
    const unsigned long long info[2] = {(unsigned long long)mode + 1, C};
    CFB_CUDA(cudaMemcpyAsync(w.info, info, sizeof(info), cudaMemcpyHostToDevice, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_components = C;
    return CFB_OK;
  });
}

extern "C" int cfb_fill_holes_graph_device(void* d_workspace, int64_t z, int64_t y, int64_t x, void* d_table, int64_t table_slots,
                                           int64_t* num_edges, void* stream) {
  return guarded([&]() -> int {
    if (!d_workspace || !d_table || !num_edges) throw std::invalid_argument("fill holes: null argument");
    fh_check_slots(table_slots);
    const Int3 sz = fh_size(z, y, x);
    const int64_t n = fh_voxels(sz);
    const FhWork w = fh_work(d_workspace, n);
    const FhTable t = fh_table(d_table, table_slots);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long h[4];
    fh_read_info(w, h, s);
    if (h[0] == CFB_FILL_BINARY + 1) throw std::invalid_argument("fill holes: binary mode needs no component graph");
    CFB_CUDA(cudaMemsetAsync(t.keys, 0, (size_t)table_slots * 8, s));
    CFB_CUDA(cudaMemsetAsync(t.info, 0, 4 * sizeof(uint32_t), s));
    launch(fh_graph_kernel, fh_grid(n), kFhThreads, 0, s, (const uint32_t*)w.comp, sz, t.keys, (unsigned long long)(table_slots - 1), t.info);
    uint32_t hi[2] = {0, 0};
    CFB_CUDA(cudaMemcpyAsync(hi, t.info, sizeof(hi), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_edges = hi[0];
    if (hi[1]) {
      set_last_error("fill holes: the pair table is too small for this many touching component pairs");
      return CFB_ERR_CAPACITY;
    }
    return CFB_OK;
  });
}

extern "C" int cfb_fill_holes_enclose(void* d_workspace, int64_t z, int64_t y, int64_t x, void* d_table, int64_t table_slots, int64_t num_edges,
                                      void* stream) {
  return guarded([&]() -> int {
    if (!d_workspace || !d_table) throw std::invalid_argument("fill holes: null argument");
    fh_check_slots(table_slots);
    if (num_edges < 0 || num_edges > table_slots) throw std::invalid_argument("fill holes: bad number of pairs");
    const FhWork w = fh_work(d_workspace, fh_voxels(fh_size(z, y, x)));
    const FhTable t = fh_table(d_table, table_slots);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long h[4];
    fh_read_info(w, h, s);
    const int32_t mode = (int32_t)h[0] - 1;
    if (mode == CFB_FILL_BINARY) throw std::invalid_argument("fill holes: binary mode needs no enclosure");
    const int64_t C = (int64_t)h[1];
    std::vector<uint8_t> flags;
    std::vector<unsigned long long> pairs;
    std::vector<uint32_t> map;
    try {
      flags.resize((size_t)C);
      pairs.resize((size_t)num_edges);
      map.resize((size_t)C);
      CFB_CUDA(cudaMemsetAsync(t.info + 2, 0, sizeof(uint32_t), s));
      launch(fh_gather_kernel, fh_grid(table_slots), kFhThreads, 0, s, (const unsigned long long*)t.keys, table_slots, t.okeys, t.info + 2);
      uint32_t got = 0;
      CFB_CUDA(cudaMemcpyAsync(&got, t.info + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaMemcpyAsync(flags.data(), w.flags, (size_t)C, cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaMemcpyAsync(pairs.data(), t.okeys, (size_t)num_edges * 8, cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaStreamSynchronize(s));
      if ((int64_t)got != num_edges) throw std::invalid_argument("fill holes: num_edges does not match the table");
      fh_enclose_host(C, flags.data(), pairs.data(), num_edges, mode, map.data());
    } catch (const std::bad_alloc&) {
      throw std::runtime_error("fill holes: the enclosure of " + std::to_string(C) + " components and " + std::to_string(num_edges) +
                               " pairs does not fit in host memory (about 40 bytes per component and 16 per pair)");
    }
    CFB_CUDA(cudaMemcpyAsync(w.rank, map.data(), (size_t)C * 4, cudaMemcpyHostToDevice, s));
    const unsigned long long done = 1ULL;
    CFB_CUDA(cudaMemcpyAsync(w.info + 3, &done, 8, cudaMemcpyHostToDevice, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    return CFB_OK;
  });
}

extern "C" int cfb_fill_holes_apply_device(const void* d_in, int32_t dtype, int64_t z, int64_t y, int64_t x, void* d_workspace, void* d_out,
                                           int64_t* fill_count, void* stream) {
  return guarded([&]() -> int {
    if (!d_in || !d_workspace || !d_out || !fill_count) throw std::invalid_argument("fill holes: null argument");
    const Int3 sz = fh_size(z, y, x);
    const int64_t n = fh_voxels(sz);
    const FhWork w = fh_work(d_workspace, n);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long h[4];
    fh_read_info(w, h, s);
    const int32_t mode = (int32_t)h[0] - 1;
    fh_check_mode(dtype, mode);
    if (mode != CFB_FILL_BINARY && !h[3]) throw std::invalid_argument("fill holes: the per-object modes apply after cfb_fill_holes_enclose");
    CFB_CUDA(cudaMemsetAsync(w.info + 2, 0, 8, s));
    if (dtype == CFB_DTYPE_U8) fh_apply<uint8_t>(d_in, d_out, mode, n, w, s);
    else if (dtype == CFB_DTYPE_F32) fh_apply<float>(d_in, d_out, mode, n, w, s);
    else if (dtype == CFB_DTYPE_U32) fh_apply<uint32_t>(d_in, d_out, mode, n, w, s);
    else fh_apply<unsigned long long>(d_in, d_out, mode, n, w, s);
    unsigned long long count = 0;
    CFB_CUDA(cudaMemcpyAsync(&count, w.info + 2, 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *fill_count = (int64_t)count;
    return CFB_OK;
  });
}
