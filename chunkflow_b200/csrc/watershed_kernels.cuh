// Device code of the `agglomerate` operator's voxel passes (the union-find they share with connected components: union_find.cuh).
// NOT a stand-alone header: segmentation.cu includes it inside the library's anonymous namespace (after `Int3` and `kT`);
// tests/host_emulation/ws_emulation.cpp compiles segmentation.cu for the host behind a one-thread CUDA shim, so that the
// kernels and their launch sequences are checked against oracle/agglomeration_oracle.py on machines without a GPU as well.
#pragma once

#include "union_find.cuh"


// ------------------------------------------------------------------------------------------
// `agglomerate` (reference plugins/agglomerate.py:8-48 -> waterz.agglomerate; waterz is NOT vendored, its published algorithm
// is restated in oracle/agglomeration_oracle.py): fragments by steepest-ascent watershed, region graph, relabel.
// Affinity layout: (3, z, y, x) float32; `flip` = 1 when the channels are stored in chunkflow's order x, y, z (the plugin's
// flip_channel, agglomerate.py:26-29) -- the kernels then read channel 2 - axis instead of copying the map.
// Direction d: 0..2 = the lower neighbour along axis d (z, y, x), 3..5 = the upper one.
// ------------------------------------------------------------------------------------------
constexpr uint32_t kWsInf = 0xFFFFFFFFu;

struct WsGeom {
  Int3 sz;
  int64_t n;        // voxels
  int64_t step[3];  // linear index step along z, y, x
};

__device__ __forceinline__ void ws_coords(int64_t i, const Int3& sz, int c[3]) {
  c[2] = (int)(i % sz.x);
  c[1] = (int)((i / sz.x) % sz.y);
  c[0] = (int)(i / ((int64_t)sz.x * sz.y));
}

__device__ __forceinline__ int64_t ws_step(const WsGeom& g, int d) { return d < 3 ? -g.step[d] : g.step[d - 3]; }

// step 1 (waterz backend/watershed.hpp "steepest ascent graph"): val[i] = bit d set when the voxel keeps its edge in
// direction d -- the edge's affinity equals the maximum of the six (which must exceed `low`) or reaches `high`; edges that
// leave the volume count as `low`.  A NaN among the six leaves the voxel without edges (numpy's max propagates NaN).
__global__ void __launch_bounds__(kT) ws_bits_kernel(const float* __restrict__ affs, WsGeom g, int flip, float low, float high,
                                                     uint32_t* __restrict__ P, uint32_t* __restrict__ val) {
  const int dim[3] = {g.sz.z, g.sz.y, g.sz.x};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
    int c[3];
    ws_coords(i, g.sz, c);
    float w[6];
    bool nan = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float* ch = affs + (int64_t)(flip ? 2 - a : a) * g.n + i;
      w[a] = c[a] > 0 ? ch[0] : low;
      w[a + 3] = c[a] < dim[a] - 1 ? ch[g.step[a]] : low;
      nan |= (w[a] != w[a]) | (w[a + 3] != w[a + 3]);
    }
    const float m = fmaxf(fmaxf(fmaxf(w[0], w[1]), fmaxf(w[2], w[3])), fmaxf(w[4], w[5]));
    uint32_t bits = 0;
    if (!nan && m > low) {
#pragma unroll
      for (int d = 0; d < 6; ++d) bits |= (uint32_t)(w[d] == m || w[d] >= high) << d;
    }
    P[i] = (uint32_t)i;
    val[i] = bits;
  }
}

// step 2: plateau corners = voxels with an edge the neighbour does not return -> distance 0; everything else "unreached"
__global__ void __launch_bounds__(kT) ws_corner_kernel(const uint32_t* __restrict__ val, WsGeom g, uint32_t* __restrict__ dist) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t bits = val[i];
    bool corner = false;
    for (int d = 0; d < 6; ++d)
      if ((bits >> d) & 1u) corner |= !((val[i + ws_step(g, d)] >> (d < 3 ? d + 3 : d - 3)) & 1u);
    dist[i] = corner ? 0u : kWsInf;
  }
}

// step 3, one breadth-first level over the two-way edges of the plateaus (a voxel that is not a corner has only two-way
// edges).  Concurrent writers store `level`, readers compare with level - 1: no hazard.
__global__ void __launch_bounds__(kT) ws_bfs_kernel(const uint32_t* __restrict__ val, WsGeom g, uint32_t* __restrict__ dist,
                                                    uint32_t level, uint32_t* __restrict__ changed) {
  bool any = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t bits = val[i];
    if (!bits || dist[i] != kWsInf) continue;
    for (int d = 0; d < 6; ++d)
      if (((bits >> d) & 1u) && dist[i + ws_step(g, d)] == level - 1u) { dist[i] = level; any = true; break; }
  }
  if (any) *changed = 1u;
}

// steps 3 + 4: every voxel reached from a corner keeps ONE edge and is united with its target; the voxels of a plateau
// without a corner (local maxima, saturated regions) keep all their edges.  Corner: the highest direction whose target
// never pointed back or is a corner at a lower raster index (what the sequential code's `to_set` ends up as); interior at
// distance L: the highest direction towards a voxel at distance L - 1 (oracle/agglomeration_oracle.py: _final_direction).
__global__ void __launch_bounds__(kT) ws_merge_kernel(const uint32_t* __restrict__ val, const uint32_t* __restrict__ dist, WsGeom g,
                                                      uint32_t* __restrict__ P) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t bits = val[i];
    if (!bits) continue;
    const uint32_t dv = dist[i];
    int fin = -1;
    for (int d = 0; d < 6; ++d) {
      if (!((bits >> d) & 1u)) continue;
      const int64_t j = i + ws_step(g, d);
      if (!val[j]) continue;  // only a voxel next to NaN affinities (no edges of its own) can be pointed at: never part of a basin
      if (dv == kWsInf) { uf_unite(P, (uint32_t)i, (uint32_t)j); continue; }
      const uint32_t dj = dist[j];
      bool cand;
      if (dv == 0u) cand = !((val[j] >> (d < 3 ? d + 3 : d - 3)) & 1u) || (d < 3 && dj == 0u);
      else cand = dj == dv - 1u;
      if (cand) fin = d;
    }
    if (fin >= 0) uf_unite(P, (uint32_t)i, (uint32_t)(i + ws_step(g, fin)));
  }
}

// ---- region graph (waterz backend/region_graph.hpp + MeanAffinityProvider): one record per pair of touching fragments, the
// sum (2^-30 fixed point: order independent) and the number of the affinities between them.  Open-addressing hash table in
// global memory (hash_table.cuh), key = (smaller id << 32 | larger id), 0 = empty slot.
#include "hash_table.cuh"

__device__ __forceinline__ long long rg_quantize(float a) {
  double v = (double)a;
  v = (v != v) ? 0.0 : fmin(fmax(v, 0.0), 1.0);
  return __double2ll_rn(v * 1073741824.0);
}

// an affinity clamped to [0, 1] in float32, NaN (and -0) as +0: the value rg_quantize quantises
__device__ __forceinline__ float rg_clamp(float a) { return a > 0.f ? fminf(a, 1.f) : 0.f; }

// kHist = false: the mean's statistics (sums, counts).  kHist = true: the first pass of the histogram region graph -- the
// same pair table, with the largest clamped face affinity per pair instead (atomicMax on the float bits: all values are
// >= +0, whose bit patterns order like the floats); `sums` and `counts` are unused and `maxbits` is written.
template <bool kHist>
__global__ void __launch_bounds__(kT) rg_accumulate_kernel(const float* __restrict__ affs, const uint32_t* __restrict__ frag, WsGeom g,
                                                           int flip, unsigned long long* __restrict__ keys,
                                                           unsigned long long* __restrict__ sums, uint32_t* __restrict__ counts,
                                                           uint32_t* __restrict__ maxbits, unsigned long long mask,
                                                           uint32_t* __restrict__ info) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t id1 = frag[i];
    if (!id1) continue;
    int c[3];
    ws_coords(i, g.sz, c);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (c[a] == 0) continue;
      const uint32_t id2 = frag[i - g.step[a]];
      if (!id2 || id2 == id1) continue;
      const unsigned long long key = ((unsigned long long)min(id1, id2) << 32) | max(id1, id2);
      const float aff = affs[(int64_t)(flip ? 2 - a : a) * g.n + i];
      const long long q = rg_quantize(aff);   // (unused, and dropped, with kHist)
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
        if constexpr (kHist) {
          const float c = rg_clamp(aff);
          uint32_t bits;
          memcpy(&bits, &c, sizeof bits);
          atomicMax(&maxbits[h], bits);
        } else {
          atomicAdd(&sums[h], (unsigned long long)q);
          atomicAdd(&counts[h], 1u);
        }
        done = true;
        break;
      }
      if (!done) info[1] = 1u;   // table too full: the host retries with a larger one
    }
  }
}

__global__ void __launch_bounds__(kT) rg_gather_kernel(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ sums,
                                                       const uint32_t* __restrict__ counts, int64_t slots, unsigned long long* __restrict__ okeys,
                                                       unsigned long long* __restrict__ osums, uint32_t* __restrict__ ocounts,
                                                       uint32_t* __restrict__ cursor) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (!k) continue;
    const uint32_t o = atomicAdd(cursor, 1u);
    okeys[o] = k; osums[o] = sums[i]; ocounts[o] = counts[i];
  }
}

// ---- histogram region graph (waterz HistogramQuantileAffinity): per pair of fragments, the number of faces whose clamped
// affinity falls in each of `bins` bins, bin = min((int)(a * bins), bins - 1) in float32.  Second pass over the faces, after
// rg_accumulate_kernel<true> built the pair table: every face finds its pair's slot and counts into a second table keyed by
// ((slot + 1) << 8 | bin) (never 0: slots are below 2^31 and bins below 256).  info[2] = entries, info[3] = overflow.
__global__ void __launch_bounds__(kT) rg_hist_kernel(const float* __restrict__ affs, const uint32_t* __restrict__ frag, WsGeom g, int flip,
                                                     const unsigned long long* __restrict__ keys, unsigned long long mask, int bins,
                                                     unsigned long long* __restrict__ hkeys, uint32_t* __restrict__ hcounts,
                                                     unsigned long long hmask, uint32_t* __restrict__ info) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t id1 = frag[i];
    if (!id1) continue;
    int c[3];
    ws_coords(i, g.sz, c);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (c[a] == 0) continue;
      const uint32_t id2 = frag[i - g.step[a]];
      if (!id2 || id2 == id1) continue;
      const unsigned long long key = ((unsigned long long)min(id1, id2) << 32) | max(id1, id2);
      unsigned long long h = rg_hash(key) & mask;
      int probe = 0;
      for (; probe < kRgMaxProbe && keys[h] != key; ++probe) {
        if (keys[h] == 0ULL) { probe = kRgMaxProbe; break; }   // not in the table: the first pass overflowed and says so
        h = (h + 1) & mask;
      }
      if (probe == kRgMaxProbe) continue;
      const int bin = min((int)__fmul_rn(rg_clamp(affs[(int64_t)(flip ? 2 - a : a) * g.n + i]), (float)bins), bins - 1);
      const unsigned long long hkey = ((h + 1ULL) << 8) | (unsigned long long)bin;
      unsigned long long s = rg_hash(hkey) & hmask;
      bool done = false;
      for (int p = 0; p < kRgMaxProbe; ++p, s = (s + 1) & hmask) {
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(hkeys + s);
        if (cur != hkey) {
          if (cur != 0ULL) continue;
          cur = atomicCAS(&hkeys[s], 0ULL, hkey);
          if (cur == 0ULL) atomicAdd(&info[2], 1u);
          else if (cur != hkey) continue;
        }
        atomicAdd(&hcounts[s], 1u);
        done = true;
        break;
      }
      if (!done) info[3] = 1u;
    }
  }
}

// compaction of the pair table: (key, max) per pair in arbitrary order, and slot_index[slot] = its position
__global__ void __launch_bounds__(kT) rg_hist_gather_pairs_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ maxbits,
                                                                  int64_t slots, unsigned long long* __restrict__ okeys,
                                                                  uint32_t* __restrict__ omax, uint32_t* __restrict__ slot_index,
                                                                  uint32_t* __restrict__ cursor) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (!k) continue;
    const uint32_t o = atomicAdd(cursor, 1u);
    okeys[o] = k; omax[o] = maxbits[i]; slot_index[i] = o;
  }
}

// compaction of the bin table: (pair position << 8 | bin, count), arbitrary order
__global__ void __launch_bounds__(kT) rg_hist_gather_bins_kernel(const unsigned long long* __restrict__ hkeys, const uint32_t* __restrict__ hcounts,
                                                                 int64_t hslots, const uint32_t* __restrict__ slot_index,
                                                                 unsigned long long* __restrict__ okeys, uint32_t* __restrict__ ocounts,
                                                                 uint32_t* __restrict__ cursor) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hslots; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = hkeys[i];
    if (!k) continue;
    const uint32_t o = atomicAdd(cursor, 1u);
    okeys[o] = ((unsigned long long)slot_index[(k >> 8) - 1] << 8) | (k & 0xFFULL);
    ocounts[o] = hcounts[i];
  }
}

__global__ void __launch_bounds__(kT) relabel_map_kernel(const uint32_t* __restrict__ labels, int64_t n, const uint32_t* __restrict__ map,
                                                         uint32_t map_size, uint32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t l = labels[i];
    out[i] = l < map_size ? map[l] : l;
  }
}

