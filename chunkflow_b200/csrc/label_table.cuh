// Device code of the segmentation clean-up (`mask-out-objects`, `remap-segmentation`, DeviceChunk.unique): the table of a
// label volume and the relabelling it plans.  NOT a stand-alone header: relabel.cu includes it inside the library's anonymous
// namespace (after `kT`); tests/host_emulation/relabel_emulation.cpp compiles relabel.cu for the host behind a one-thread,
// one-lane CUDA shim (EV_WARP = 1), so that the kernels and their launch sequences are checked against oracle/relabel_oracle.py
// on machines without a GPU.
//
// One table (state_table.cuh: any uint64 is a legal id), a power of two of slots:
//   id -> (voxel count, linear index of the id's first voxel in raster order, new value)
// Three steps, each reading the volume at most once:
//   count   lt_count_kernel: one atomicAdd and one atomicMin per RUN of equal ids, not per voxel
//   plan    lt_keep / lt_decide / lt_block_count / (cc_scan_blocks_kernel) / lt_rank: every entry's new value, from the table
//           alone: 0 for dust and for ids outside the keep-list, else the id itself or, when renumbering, 1 + base id + the
//           rank of its first voxel among the survivors' first voxels
//   apply   lt_apply_kernel: one table probe per run, one write per voxel
//
// Runs: a lane loads 16 bytes (V = 2, 4 or 16 consecutive ids), a warp 32 * V consecutive ids.  A run is owned by the lane
// in which it starts; it extends over the following lanes that hold nothing but its id and into the leading ids of the first
// lane that does not (lt_runs).  A one-lane warp keeps the in-lane part of this logic.
#pragma once

#include "state_table.cuh"

#if EV_WARP == 32
__device__ __forceinline__ unsigned long long lt_shfl(unsigned long long v, int src) { return __shfl_sync(0xffffffffu, v, src); }
#else
inline unsigned long long lt_shfl(unsigned long long v, int) { return v; }
#endif

// statistics block at the start of the workspace (uint64 words)
enum LtStat {
  kLtLabels = 0,     // entries of the table (0 included when it occurs)
  kLtOverflow,       // != 0: the table is too full
  kLtDust,           // plan: entries with count <= the dust threshold (0 included), what mask_fragments reports
  kLtSurvivors,      // plan: non-zero ids whose new value is not 0
  kLtMax,            // plan without renumbering: the largest new value
  kLtRenumbered,     // plan: != 0 when the new values are ranks (they need a uint64 output)
  kLtPlanned,        // plan: != 0 once every entry has its new value
  kLtMissing,        // apply: != 0 when the volume holds an id the table does not
  kLtStatWords = 8
};

constexpr int kLtBlockWords = 4 * EV_WARP;   // flag words (32 voxels each) per scan block: 4096 voxels on the device

struct LtTable {
  unsigned long long* stats;   // kLtStatWords
  unsigned long long *keys, *newval;
  uint32_t *state, *count, *first, *flags;   // flags: bit 0 on the keep-list, bit 1 to be ranked
  unsigned long long mask;     // slots - 1
};

// slot of an id of a complete table, -1 when it is not there
__device__ __forceinline__ long long lt_find(const LtTable& t, unsigned long long id) {
  unsigned long long h = rg_hash(id) & t.mask;
  for (int probe = 0; probe < kRgMaxProbe; ++probe, h = (h + 1) & t.mask) {
    if (t.state[h] != 2u) return -1;
    if (t.keys[h] == id) return (long long)h;
  }
  return -1;
}

// ids are held in 32- or 64-bit registers whatever their width in memory (byte-typed arrays end up in local memory)
template <typename T> struct LtReg { typedef uint32_t type; };
template <> struct LtReg<uint64_t> { typedef unsigned long long type; };

// the 16 bytes of a vector load or store as ids (shifts on the four words: everything stays in registers)
__device__ __forceinline__ uint32_t lt_word(const uint4& q, int k) { return k == 0 ? q.x : k == 1 ? q.y : k == 2 ? q.z : q.w; }

template <typename T>
__device__ __forceinline__ typename LtReg<T>::type lt_unpack(const uint4& q, int e) {
  if constexpr (sizeof(T) == 1) return (lt_word(q, e >> 2) >> (8 * (e & 3))) & 0xffu;
  else if constexpr (sizeof(T) == 4) return lt_word(q, e);
  else return (unsigned long long)lt_word(q, 2 * e) | ((unsigned long long)lt_word(q, 2 * e + 1) << 32);
}

template <typename T, int V>
__device__ __forceinline__ uint4 lt_pack(const typename LtReg<T>::type (&o)[V], int k) {   // ids [k * 16 / sizeof(T), (k + 1) * 16 / sizeof(T))
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if constexpr (sizeof(T) == 1) {
      const int b = 16 * k + 4 * j;
      w[j] = (o[b] & 0xffu) | ((o[b + 1] & 0xffu) << 8) | ((o[b + 2] & 0xffu) << 16) | (o[b + 3] << 24);
    } else if constexpr (sizeof(T) == 4) {
      w[j] = (uint32_t)o[4 * k + j];
    } else {
      w[j] = (uint32_t)((unsigned long long)o[2 * k + (j >> 1)] >> (32 * (j & 1)));
    }
  }
  uint4 q;
  q.x = w[0]; q.y = w[1]; q.z = w[2]; q.w = w[3];
  return q;
}

// V consecutive ids from i0 (one 16-byte load when they all exist) -> how many exist
template <typename T, int V>
__device__ __forceinline__ int lt_load(const T* p, int64_t i0, int64_t n, typename LtReg<T>::type (&v)[V]) {
  if (i0 + V <= n) {
    const uint4 q = *reinterpret_cast<const uint4*>(p + i0);
#pragma unroll
    for (int e = 0; e < V; ++e) v[e] = lt_unpack<T>(q, e);
    return V;
  }
  int cnt = 0;
#pragma unroll
  for (int e = 0; e < V; ++e) {
    v[e] = 0;
    if (i0 + e < n) { v[e] = p[i0 + e]; cnt = e + 1; }
  }
  return cnt;
}

struct LtRuns {
  int lead;        // ids at the start of the lane that equal its first id
  bool joins;      // the leading run started in an earlier lane
  uint32_t brk;    // lanes that are NOT a mere continuation of an earlier lane's run
  uint32_t ext;    // ids beyond this lane that belong to the run that is open at its end
};

template <typename T, int V>
__device__ __forceinline__ LtRuns lt_runs(const T (&v)[V], int cnt, int lane) {   // T: the ids' register type
  LtRuns r;
  r.lead = 0;
  bool eq = true;
  T last = v[0];
#pragma unroll
  for (int e = 0; e < V; ++e) {
    eq = eq && e < cnt && v[e] == v[0];
    r.lead += eq ? 1 : 0;
    if (e < cnt) last = v[e];
  }
  const unsigned long long prev_last = ev_shfl_up((unsigned long long)last);
  r.joins = lane > 0 && cnt > 0 && prev_last == (unsigned long long)v[0];   // cnt > 0: the previous lane is complete
  const bool cont = r.joins && r.lead == V;
  r.brk = ev_ballot(!cont);
  const uint32_t above = r.brk & (uint32_t)(~0ULL << (lane + 1));
  const int j = above ? __ffs((int)above) - 1 : EV_WARP;                    // the lane in which the open run ends
  const unsigned long long jl = lt_shfl(r.joins ? (unsigned long long)r.lead : 0ULL, j & (EV_WARP - 1));
  r.ext = (uint32_t)((j - lane - 1) * V) + (j < EV_WARP ? (uint32_t)jl : 0u);
  return r;
}

__device__ __forceinline__ void lt_add(const LtTable& t, unsigned long long id, uint32_t len, uint32_t first) {
  bool inserted = false;
  const long long h = ev_slot<false>(t.state, t.keys, nullptr, id, 0ULL, t.mask, &inserted);
  if (h < 0) { t.stats[kLtOverflow] = 1ULL; return; }   // table too full: the host retries with a larger one
  if (inserted) atomicAdd(&t.stats[kLtLabels], 1ULL);
  atomicAdd(&t.count[h], len);
  atomicMin(&t.first[h], first);
}

// ---- count pass ----
template <typename T>
__global__ void __launch_bounds__(kT, 4) lt_count_kernel(const T* __restrict__ labels, int64_t n, LtTable t) {
  constexpr int V = 16 / (int)sizeof(T);
  const int lane = ev_lane();
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / EV_WARP;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * V;   // ids per sweep of the whole grid
  for (int64_t base = warp * EV_WARP * V; base < n; base += stride) {   // warp-uniform: every lane reaches the shuffles
    const int64_t i0 = base + (int64_t)lane * V;
    typename LtReg<T>::type v[V];
    const int cnt = lt_load<T, V>(labels, i0, n, v);
    const LtRuns r = lt_runs(v, cnt, lane);
    auto cur = v[0];
    int s = 0;
#pragma unroll
    for (int e = 1; e <= V; ++e) {
      const auto next = v[e < V ? e : 0];
      if (e > cnt || (e < cnt && next == cur)) continue;
      if (!(s == 0 && r.joins))                                   // the run [s, e) starts in this lane
        lt_add(t, (unsigned long long)cur, (uint32_t)(e - s) + (e == V ? r.ext : 0u), (uint32_t)(i0 + s));
      cur = next;
      s = e;
    }
  }
}

// ---- plan ----
__global__ void __launch_bounds__(kT) lt_keep_kernel(const unsigned long long* __restrict__ keep, int64_t num_keep, LtTable t) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_keep; i += stride) {
    const long long h = lt_find(t, keep[i]);
    if (h >= 0) t.flags[h] = 1u;   // ids that do not occur are ignored
  }
}

__global__ void __launch_bounds__(kT) lt_decide_kernel(LtTable t, int use_dust, long long dust_threshold, int use_keep, int renumber,
                                                       uint32_t* __restrict__ bits) {
  unsigned long long dust = 0, survivors = 0;
  const int64_t slots = (int64_t)t.mask + 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride) {
    if (t.state[s] != 2u) continue;
    const bool dusty = use_dust && (long long)t.count[s] <= dust_threshold;   // `<=`: reference chunk/segmentation.py:88
    uint32_t f = t.flags[s] & 1u;
    const unsigned long long nv = (dusty || (use_keep && !f)) ? 0ULL : t.keys[s];
    dust += dusty ? 1ULL : 0ULL;
    if (nv != 0ULL) {
      ++survivors;
      if (renumber) {
        f |= 2u;
        const uint32_t i = t.first[s];
        atomicOr(&bits[i >> 5], 1u << (i & 31u));
      } else {
        atomicMax(&t.stats[kLtMax], nv);
      }
    }
    t.newval[s] = nv;
    t.flags[s] = f;
  }
  dust = ev_warp_sum(dust);
  survivors = ev_warp_sum(survivors);
  if (ev_lane() == 0 && dust) atomicAdd(&t.stats[kLtDust], dust);
  if (ev_lane() == 0 && survivors) atomicAdd(&t.stats[kLtSurvivors], survivors);
}

// first level of the ranking: flags set per block of kLtBlockWords words, one warp per block
__global__ void __launch_bounds__(kT) lt_block_count_kernel(const uint32_t* __restrict__ bits, int64_t nblocks,
                                                            uint32_t* __restrict__ block_count) {
  const int lane = ev_lane();
  const int64_t warps = (int64_t)gridDim.x * blockDim.x / EV_WARP;
  for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / EV_WARP; b < nblocks; b += warps) {
    unsigned long long c = 0;
#pragma unroll
    for (int k = 0; k < kLtBlockWords / EV_WARP; ++k) c += (unsigned long long)__popc(bits[b * kLtBlockWords + k * EV_WARP + lane]);
    c = ev_warp_sum(c);
    if (lane == 0) block_count[b] = (uint32_t)c;
  }
}

// third level: new value of a ranked entry = flags before its first voxel (block base + inside the block) + 1 + base id
__global__ void __launch_bounds__(kT) lt_rank_kernel(LtTable t, const uint32_t* __restrict__ bits, const uint32_t* __restrict__ block_base,
                                                     unsigned long long base_id) {
  const int64_t slots = (int64_t)t.mask + 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride) {
    if (t.state[s] != 2u || !(t.flags[s] & 2u)) continue;
    const uint32_t i = t.first[s], w = i >> 5;
    const uint32_t b = w / (uint32_t)kLtBlockWords;
    unsigned long long r = block_base[b];
    for (uint32_t k = b * (uint32_t)kLtBlockWords; k < w; ++k) r += (unsigned long long)__popc(bits[k]);
    r += (unsigned long long)__popc(bits[w] & ((1u << (i & 31u)) - 1u));
    t.newval[s] = r + 1ULL + base_id;
  }
}

// ---- apply pass (out may be in when the types are equal: a lane writes only what it has read) ----
template <typename TI, typename TO>
__global__ void __launch_bounds__(kT, 4) lt_apply_kernel(const TI* in, int64_t n, LtTable t, TO* out) {
  constexpr int V = 16 / (int)sizeof(TI);
  const int lane = ev_lane();
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / EV_WARP;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * V;
  for (int64_t base = warp * EV_WARP * V; base < n; base += stride) {
    const int64_t i0 = base + (int64_t)lane * V;
    typename LtReg<TI>::type v[V];
    const int cnt = lt_load<TI, V>(in, i0, n, v);
    const LtRuns r = lt_runs(v, cnt, lane);
    typedef typename LtReg<TO>::type RO;
    RO o[V];
    auto cur = v[0];
    unsigned long long cur_new = 0ULL;   // of a leading run that started earlier: filled in below
#pragma unroll
    for (int e = 0; e < V; ++e) {
      if (e < cnt && (e == 0 ? !r.joins : v[e] != cur)) {   // a run starts here: one probe
        cur = v[e];
        const long long h = lt_find(t, (unsigned long long)cur);
        if (h < 0) t.stats[kLtMissing] = 1ULL;
        cur_new = h < 0 ? 0ULL : t.newval[h];
      }
      o[e] = (RO)cur_new;
    }
    // the value of a joined leading run comes from the nearest earlier lane that looked one up for its last run
    const uint32_t below = r.brk & ((1u << lane) - 1u);
    const unsigned long long inherited = lt_shfl(cur_new, below ? 31 - __clz((int)below) : 0);
    if (r.joins) {
#pragma unroll
      for (int e = 0; e < V; ++e)
        if (e < r.lead) o[e] = (RO)inherited;
    }
    if (cnt == V) {
      constexpr int Q = V * (int)sizeof(TO) / 16;
#pragma unroll
      for (int k = 0; k < Q; ++k) reinterpret_cast<uint4*>(out + i0)[k] = lt_pack<TO, V>(o, k);
    } else {
#pragma unroll
      for (int e = 0; e < V; ++e)
        if (e < cnt) out[i0 + e] = (TO)o[e];
    }
  }
}
