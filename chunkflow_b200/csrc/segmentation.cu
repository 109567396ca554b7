// `connected-components` on the device (SURVEY.md section 8 f4): the operator that follows `inference` in the reference's
// README pipeline.  Reference: Chunk.connected_component (chunkflow/chunk/base.py:128-137) -> Chunk.threshold (:728-737) ->
// cc3d.connected_components(seg, connectivity) -- cc3d is a third-party package that is NOT vendored in the reference tree
// (requirements.txt: connected-components-3d); its published behaviour, restated in oracle/segmentation_oracle.py:
//   * voxels are connected when they are 6 / 18 / 26-neighbours AND carry the same non-zero value (multi-label input),
//   * 0 is background and stays 0,
//   * output labels are 1 .. N, numbered in the order in which the components are first met in a raster scan of the
//     memory (x fastest, then y, then z for a C-order (z, y, x) array).
//
// Kernels (HBM / atomic bound, no tensor work): label-equivalence union-find over the voxels' linear indices
//   init      P[i] = i
//   merge     for every foreground voxel, unite with the backward half of its neighbourhood (3 / 9 / 13 neighbours)
//             that carries the same value: root search + atomicMin on the larger root (lock-free, any order)
//   flatten   P[i] = root(i): the root of a component is its smallest linear index = its first voxel in raster order
//   rank      exclusive prefix sum of the root flags in raster order (two-level scan) -> label of a root = rank + 1
//   relabel   out[i] = rank[P[i]] + 1 for foreground, 0 for background
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <type_traits>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"
#include "edge_sort.h"

namespace cfb {
namespace {

constexpr int kT = 256;
constexpr int kScanBlock = 4096;  // voxels per scan block (16 per thread)

template <typename T>
__device__ __forceinline__ uint32_t fg_value(const T* __restrict__ in, int64_t i, float threshold, bool use_threshold) {
  if constexpr (sizeof(T) == 4 && !std::is_integral<T>::value) {
    return in[i] > threshold ? 1u : 0u;  // Chunk.threshold: array > threshold (base.py:729)
  } else {
    (void)threshold; (void)use_threshold;
    return (uint32_t)in[i];
  }
}

#include "watershed_kernels.cuh"  // union-find helpers + the watershed / region-graph / relabel kernels

template <typename T>
__global__ void __launch_bounds__(kT) cc_init_kernel(const T* __restrict__ in, uint32_t* __restrict__ P, uint32_t* __restrict__ val,
                                                     int64_t n, float threshold) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    P[i] = (uint32_t)i;
    val[i] = fg_value(in, i, threshold, true);
  }
}

// backward half of the 26-neighbourhood, ordered so that the first 3 are the face neighbours (6-connectivity), the first 9
// the face + edge neighbours (18) and all 13 the full neighbourhood (26)
__constant__ int kNb[13][3] = {{0, 0, -1}, {0, -1, 0}, {-1, 0, 0},
                               {0, -1, -1}, {0, -1, 1}, {-1, 0, -1}, {-1, 0, 1}, {-1, -1, 0}, {-1, 1, 0},
                               {-1, -1, -1}, {-1, -1, 1}, {-1, 1, -1}, {-1, 1, 1}};

__global__ void __launch_bounds__(kT) cc_merge_kernel(const uint32_t* __restrict__ val, uint32_t* __restrict__ P, Int3 sz, int nnb) {
  const int64_t n = (int64_t)sz.z * sz.y * sz.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t v = val[i];
    if (!v) continue;
    const int x = (int)(i % sz.x), y = (int)((i / sz.x) % sz.y), z = (int)(i / ((int64_t)sz.x * sz.y));
    for (int k = 0; k < nnb; ++k) {
      const int zz = z + kNb[k][0], yy = y + kNb[k][1], xx = x + kNb[k][2];
      if (zz < 0 || yy < 0 || yy >= sz.y || xx < 0 || xx >= sz.x) continue;
      const int64_t j = ((int64_t)zz * sz.y + yy) * sz.x + xx;
      if (val[j] == v) uf_unite(P, (uint32_t)i, (uint32_t)j);
    }
  }
}

// flatten + per-block count of roots
__global__ void __launch_bounds__(kT) cc_flatten_count_kernel(const uint32_t* __restrict__ val, uint32_t* __restrict__ P, int64_t n,
                                                              uint32_t* __restrict__ block_count) {
  __shared__ uint32_t s_count;
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kScanBlock;
  uint32_t mine = 0;
  for (int k = 0; k < kScanBlock / kT; ++k) {
    const int64_t i = base + k * kT + threadIdx.x;
    if (i < n && val[i]) {
      const uint32_t r = uf_find(P, (uint32_t)i);
      P[i] = r;   // (roots keep P[r] == r; concurrent readers only ever see an ancestor)
      mine += r == (uint32_t)i;
    }
  }
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_count, mine);
  __syncthreads();
  if (threadIdx.x == 0) block_count[blockIdx.x] = s_count;
}

// exclusive scan of the block counts by ONE block (sequential chunks of 1024 with a carry), total -> *num_labels
__global__ void __launch_bounds__(1024) cc_scan_blocks_kernel(uint32_t* __restrict__ block_count, int64_t nblocks, uint32_t* __restrict__ num_labels) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = 0; base < nblocks; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const uint32_t v = i < nblocks ? block_count[i] : 0u;
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_warp[lane];
      for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
      s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const uint32_t before = s_carry + (warp ? s_warp[warp - 1] : 0u) + incl - v;
    if (i < nblocks) block_count[i] = before;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = before + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *num_labels = s_carry;
}

// rank of every root inside its block (raster order) + the block's base -> rank[root]
__global__ void __launch_bounds__(kT) cc_rank_kernel(const uint32_t* __restrict__ val, const uint32_t* __restrict__ P, int64_t n,
                                                     const uint32_t* __restrict__ block_base, uint32_t* __restrict__ rank) {
  __shared__ uint32_t s_warp[kT / 32];
  __shared__ uint32_t s_running;
  if (threadIdx.x == 0) s_running = block_base[blockIdx.x];
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kScanBlock;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = 0; k < kScanBlock / kT; ++k) {   // chunk k holds 256 CONSECUTIVE voxels: raster order is preserved
    const int64_t i = base + k * kT + threadIdx.x;
    const bool root = i < n && val[i] && P[i] == (uint32_t)i;
    const uint32_t ballot = __ballot_sync(0xffffffffu, root);
    const uint32_t in_warp = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    uint32_t before = s_running;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    if (root) rank[i] = before + in_warp;
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < kT / 32; ++w) t += s_warp[w]; s_running += t; }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kT) cc_relabel_kernel(const uint32_t* __restrict__ val, const uint32_t* __restrict__ P,
                                                        const uint32_t* __restrict__ rank, uint32_t* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = val[i] ? rank[P[i]] + 1u : 0u;
}

WsGeom ws_geom(int64_t z, int64_t y, int64_t x) {
  if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX) throw std::invalid_argument("bad volume size");
  WsGeom g;
  g.sz = Int3{(int)z, (int)y, (int)x};
  g.n = z * y * x;
  if (g.n >= (int64_t)UINT32_MAX) throw std::invalid_argument("more than 2^32 - 1 voxels");
  g.step[0] = y * x; g.step[1] = x; g.step[2] = 1;
  return g;
}

template <typename F>
int guarded_seg(F&& f) {
  try {
    return f();
  } catch (const std::invalid_argument& ex) {
    set_last_error(ex.what());
    return CFB_ERR_INVALID_ARGUMENT;
  } catch (const CudaError& ex) {
    set_last_error(ex.what());
    return CFB_ERR_CUDA;
  } catch (const std::exception& ex) {
    set_last_error(ex.what());
    return CFB_ERR_UNSUPPORTED;
  }
}

int grid_for(int64_t items) {
  int64_t b = ceil_div64(items, kT);
  return (int)std::max<int64_t>(1, std::min<int64_t>(b, 132 * 16));
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_connected_components_device(const void* d_in, int32_t in_dtype, int64_t z, int64_t y, int64_t x, float threshold,
                                               int32_t connectivity, uint32_t* d_labels, void* d_workspace, uint32_t* num_labels,
                                               void* stream) {
  try {
    if (!d_in || !d_labels || !d_workspace) throw std::invalid_argument("null argument");
    if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX) throw std::invalid_argument("bad volume size");
    const int64_t n = z * y * x;
    if (n >= (int64_t)UINT32_MAX) throw std::invalid_argument("connected components: more than 2^32 - 1 voxels");
    int nnb;
    if (connectivity == 6) nnb = 3; else if (connectivity == 18) nnb = 9; else if (connectivity == 26) nnb = 13;
    else throw std::invalid_argument("connectivity must be 6, 18 or 26 (cc3d)");
    cudaStream_t s = (cudaStream_t)stream;
    const Int3 sz{(int)z, (int)y, (int)x};
    // workspace: P (n) | val (n) | rank (n, written at root positions only) | block counts (ceil(n / 4096)) | label count (1)
    uint32_t* P = static_cast<uint32_t*>(d_workspace);
    uint32_t* val = P + n;
    uint32_t* rank = val + n;
    const int64_t nblocks = ceil_div64(n, kScanBlock);
    uint32_t* block_count = rank + n;
    uint32_t* d_num = block_count + nblocks;
    if (in_dtype == CFB_DTYPE_U8) cc_init_kernel<uint8_t><<<grid_for(n), kT, 0, s>>>((const uint8_t*)d_in, P, val, n, 0.f);
    else if (in_dtype == CFB_DTYPE_U32) cc_init_kernel<uint32_t><<<grid_for(n), kT, 0, s>>>((const uint32_t*)d_in, P, val, n, 0.f);
    else if (in_dtype == CFB_DTYPE_F32) cc_init_kernel<float><<<grid_for(n), kT, 0, s>>>((const float*)d_in, P, val, n, threshold);
    else throw std::invalid_argument("connected components: input dtype must be uint8, uint32 or float32 (with a threshold)");
    CFB_LAUNCH_CHECK();
    cc_merge_kernel<<<grid_for(n), kT, 0, s>>>(val, P, sz, nnb);
    CFB_LAUNCH_CHECK();
    cc_flatten_count_kernel<<<(unsigned)nblocks, kT, 0, s>>>(val, P, n, block_count);
    CFB_LAUNCH_CHECK();
    cc_scan_blocks_kernel<<<1, 1024, 0, s>>>(block_count, nblocks, d_num);
    CFB_LAUNCH_CHECK();
    cc_rank_kernel<<<(unsigned)nblocks, kT, 0, s>>>(val, P, n, block_count, rank);
    CFB_LAUNCH_CHECK();
    cc_relabel_kernel<<<grid_for(n), kT, 0, s>>>(val, P, rank, d_labels, n);
    CFB_LAUNCH_CHECK();
    if (num_labels) {
      CFB_CUDA(cudaMemcpyAsync(num_labels, d_num, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaStreamSynchronize(s));
    }
    return CFB_OK;
  } catch (const std::invalid_argument& ex) {
    set_last_error(ex.what());
    return CFB_ERR_INVALID_ARGUMENT;
  } catch (const CudaError& ex) {
    set_last_error(ex.what());
    return CFB_ERR_CUDA;
  } catch (const std::exception& ex) {
    set_last_error(ex.what());
    return CFB_ERR_UNSUPPORTED;
  }
}

extern "C" int64_t cfb_connected_components_workspace(int64_t z, int64_t y, int64_t x) {
  if (z <= 0 || y <= 0 || x <= 0) return 0;
  const int64_t n = z * y * x;
  return (3 * n + ceil_div64(n, kScanBlock) + 1) * (int64_t)sizeof(uint32_t);
}

// ---- watershed fragments ------------------------------------------------------------------
extern "C" int64_t cfb_watershed_workspace(int64_t z, int64_t y, int64_t x) {
  if (z <= 0 || y <= 0 || x <= 0) return 0;
  const int64_t n = z * y * x;   // the connected-components workspace + the plateau distances + one flag
  return cfb_connected_components_workspace(z, y, x) + (n + 1) * (int64_t)sizeof(uint32_t);
}

extern "C" int cfb_watershed_device(const float* d_affs, int32_t flip_channel, int64_t z, int64_t y, int64_t x, float aff_threshold_low,
                                    float aff_threshold_high, uint32_t* d_fragments, void* d_workspace, uint32_t* num_fragments,
                                    void* stream) {
  return guarded_seg([&]() -> int {
    if (!d_affs || !d_fragments || !d_workspace) throw std::invalid_argument("watershed: null argument");
    if (!(aff_threshold_low < aff_threshold_high)) throw std::invalid_argument("watershed: need aff_threshold_low < aff_threshold_high");
    const WsGeom g = ws_geom(z, y, x);
    const int64_t n = g.n;
    cudaStream_t s = (cudaStream_t)stream;
    uint32_t* P = static_cast<uint32_t*>(d_workspace);
    uint32_t* val = P + n;
    uint32_t* rank = val + n;
    const int64_t nblocks = ceil_div64(n, kScanBlock);
    uint32_t* block_count = rank + n;
    uint32_t* d_num = block_count + nblocks;
    uint32_t* dist = d_num + 1;
    uint32_t* d_changed = dist + n;
    const int grid = grid_for(n);
    ws_bits_kernel<<<grid, kT, 0, s>>>(d_affs, g, flip_channel ? 1 : 0, aff_threshold_low, aff_threshold_high, P, val);
    CFB_LAUNCH_CHECK();
    ws_corner_kernel<<<grid, kT, 0, s>>>(val, g, dist);
    CFB_LAUNCH_CHECK();
    // breadth-first levels in batches of 8 launches per look at the flag (a level without news ends the search; the
    // remaining launches of its batch find nothing)
    uint32_t level = 1;
    for (;;) {
      CFB_CUDA(cudaMemsetAsync(d_changed, 0, sizeof(uint32_t), s));
      for (int k = 0; k < 8; ++k, ++level) {
        ws_bfs_kernel<<<grid, kT, 0, s>>>(val, g, dist, level, d_changed);
        CFB_LAUNCH_CHECK();
      }
      uint32_t changed = 0;
      CFB_CUDA(cudaMemcpyAsync(&changed, d_changed, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaStreamSynchronize(s));
      if (!changed) break;
      if (level > 0x7FFFFFF0u) throw std::runtime_error("watershed: plateau search did not end");
    }
    ws_merge_kernel<<<grid, kT, 0, s>>>(val, dist, g, P);
    CFB_LAUNCH_CHECK();
    cc_flatten_count_kernel<<<(unsigned)nblocks, kT, 0, s>>>(val, P, n, block_count);
    CFB_LAUNCH_CHECK();
    cc_scan_blocks_kernel<<<1, 1024, 0, s>>>(block_count, nblocks, d_num);
    CFB_LAUNCH_CHECK();
    cc_rank_kernel<<<(unsigned)nblocks, kT, 0, s>>>(val, P, n, block_count, rank);
    CFB_LAUNCH_CHECK();
    cc_relabel_kernel<<<grid, kT, 0, s>>>(val, P, rank, d_fragments, n);
    CFB_LAUNCH_CHECK();
    if (num_fragments) {
      CFB_CUDA(cudaMemcpyAsync(num_fragments, d_num, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      CFB_CUDA(cudaStreamSynchronize(s));
    }
    return CFB_OK;
  });
}

// ---- region graph -------------------------------------------------------------------------
// workspace: table keys | table sums | compact keys | compact sums (8 B each) | table counts | compact counts | info[4] (4 B each)
extern "C" int64_t cfb_region_graph_workspace(int64_t table_slots) {
  if (table_slots <= 0) return 0;
  return table_slots * (4 * 8 + 2 * 4) + 4 * (int64_t)sizeof(uint32_t);
}

extern "C" int cfb_region_graph_device(const float* d_affs, int32_t flip_channel, const uint32_t* d_fragments, int64_t z, int64_t y,
                                       int64_t x, void* d_workspace, int64_t table_slots, int64_t* num_edges, void* stream) {
  return guarded_seg([&]() -> int {
    if (!d_affs || !d_fragments || !d_workspace || !num_edges) throw std::invalid_argument("region graph: null argument");
    if (table_slots < 2 || (table_slots & (table_slots - 1)) || table_slots >= ((int64_t)1 << 31))
      throw std::invalid_argument("region graph: table_slots must be a power of two below 2^31");
    const WsGeom g = ws_geom(z, y, x);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* keys = static_cast<unsigned long long*>(d_workspace);
    unsigned long long* sums = keys + table_slots;
    uint32_t* counts = reinterpret_cast<uint32_t*>(keys + 4 * table_slots);
    uint32_t* info = counts + 2 * table_slots;
    CFB_CUDA(cudaMemsetAsync(keys, 0, (size_t)table_slots * 16, s));     // keys + sums
    CFB_CUDA(cudaMemsetAsync(counts, 0, (size_t)table_slots * 4, s));
    CFB_CUDA(cudaMemsetAsync(info, 0, 4 * sizeof(uint32_t), s));
    rg_accumulate_kernel<<<grid_for(g.n), kT, 0, s>>>(d_affs, d_fragments, g, flip_channel ? 1 : 0, keys, sums, counts,
                                                     (unsigned long long)(table_slots - 1), info);
    CFB_LAUNCH_CHECK();
    uint32_t h_info[2] = {0, 0};
    CFB_CUDA(cudaMemcpyAsync(h_info, info, sizeof(h_info), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_edges = h_info[0];
    if (h_info[1]) {
      set_last_error("region graph: the hash table is too small for this many fragment pairs");
      return CFB_ERR_CAPACITY;
    }
    return CFB_OK;
  });
}

extern "C" int cfb_region_graph_read(void* d_workspace, int64_t table_slots, int64_t num_edges, uint32_t* h_u, uint32_t* h_v,
                                     uint64_t* h_sum_fixed, uint32_t* h_count, void* stream) {
  return guarded_seg([&]() -> int {
    if (!d_workspace || table_slots < 2 || num_edges < 0 || num_edges > table_slots) throw std::invalid_argument("region graph read: bad argument");
    if (num_edges == 0) return CFB_OK;
    if (!h_u || !h_v || !h_sum_fixed || !h_count) throw std::invalid_argument("region graph read: null output");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* keys = static_cast<unsigned long long*>(d_workspace);
    unsigned long long* sums = keys + table_slots;
    unsigned long long* okeys = sums + table_slots;
    unsigned long long* osums = okeys + table_slots;
    uint32_t* counts = reinterpret_cast<uint32_t*>(keys + 4 * table_slots);
    uint32_t* ocounts = counts + table_slots;
    uint32_t* cursor = ocounts + table_slots + 2;   // info[2]
    CFB_CUDA(cudaMemsetAsync(cursor, 0, sizeof(uint32_t), s));
    rg_gather_kernel<<<grid_for(table_slots), kT, 0, s>>>(keys, sums, counts, table_slots, okeys, osums, ocounts, cursor);
    CFB_LAUNCH_CHECK();
    std::vector<unsigned long long> k((size_t)num_edges), sm((size_t)num_edges);
    std::vector<uint32_t> ct((size_t)num_edges);
    uint32_t got = 0;
    CFB_CUDA(cudaMemcpyAsync(&got, cursor, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(k.data(), okeys, (size_t)num_edges * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(sm.data(), osums, (size_t)num_edges * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(ct.data(), ocounts, (size_t)num_edges * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if ((int64_t)got != num_edges) throw std::invalid_argument("region graph read: num_edges does not match the table");
    std::vector<uint32_t> order;
    sorted_edge_order(k.data(), k.size(), order);   // the gather order is arbitrary
    for (size_t i = 0; i < order.size(); ++i) {
      const uint32_t o = order[i];
      h_u[i] = (uint32_t)(k[o] >> 32);
      h_v[i] = (uint32_t)(k[o] & 0xFFFFFFFFULL);
      h_sum_fixed[i] = sm[o];
      h_count[i] = ct[o];
    }
    return CFB_OK;
  });
}

extern "C" int cfb_relabel_device(const uint32_t* d_labels, int64_t n, const uint32_t* d_map, int64_t map_size, uint32_t* d_out,
                                  void* stream) {
  return guarded_seg([&]() -> int {
    if (!d_labels || !d_map || !d_out || n < 0 || map_size < 0 || map_size > (int64_t)UINT32_MAX) throw std::invalid_argument("relabel: bad argument");
    if (n == 0) return CFB_OK;
    relabel_map_kernel<<<grid_for(n), kT, 0, (cudaStream_t)stream>>>(d_labels, n, d_map, (uint32_t)map_size, d_out);
    CFB_LAUNCH_CHECK();
    return CFB_OK;
  });
}
