// Device code of `evaluate-segmentation`: the contingency table of two label volumes and the statistics the five scores
// need.  NOT a stand-alone header: evaluate.cu includes it inside the library's anonymous namespace (after `kT`);
// tests/host_emulation/evaluate_emulation.cpp includes the same text behind a one-thread, one-lane CUDA shim (it defines
// EV_WARP = 1 and the ev_* warp helpers first), so that the kernels' logic is checked against oracle/evaluation_oracle.py on
// machines without a GPU as well.
//
// Every uint64 value is a legal label (0 and 2^64 - 1 included), so no key value can mark an empty slot: each slot carries
// a state word (0 empty, 1 being written, 2 ready) and the keys are written by the thread that claimed the slot.
//
// Three tables of the same number of slots (a power of two):
//   pair  (seg id, gt id) -> voxel count c                            built from the voxels (ev_pairs_kernel)
//   row   seg id -> (sum of c, sum of c over gt id != 0)               built from the pair table (ev_margins_kernel)
//   col   gt id  -> (sum of c, sum of c over seg id != 0)              built from the pair table (ev_margins_kernel)
// A table never holds more keys than the pair table, so one slot count serves all three.
//
// Determinism: every statistic is a sum of integers (atomics in any order give the same result), including the fp64
// entropy sums: each term c * log2(c) is a double >= 2 (or 0), hence a multiple of 2^-51 below 2^37; it is split into its
// integer part and two 26-bit limbs of its fraction, which are summed exactly in uint64 and composed once on the host.
#pragma once

#include "hash_table.cuh"

#ifndef EV_WARP
#define EV_WARP 32
__device__ __forceinline__ int ev_lane() { return (int)(threadIdx.x & 31u); }
__device__ __forceinline__ unsigned long long ev_shfl_up(unsigned long long v) { return __shfl_up_sync(0xffffffffu, v, 1); }
__device__ __forceinline__ uint32_t ev_ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ unsigned long long ev_warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif

// statistics block at the start of the workspace (uint64 words)
enum EvStat {
  kEvN = 0,          // voxels
  kEvS1,             // sum of c^2 over all pairs
  kEvS2,             // sum of row^2 (all voxels)
  kEvS3,             // sum of col^2 (all voxels)
  kEvNBoth,          // voxels with both ids != 0
  kEvSegIds,         // distinct non-zero seg ids
  kEvGtIds,          // distinct non-zero gt ids
  kEvPairs,          // entries of the pair table
  kEvRows,           // entries of the row table (0 included)
  kEvCols,           // entries of the col table
  kEvOverflow,       // != 0: some table is too full
  kEvXlC = 11,       // 3 limbs: sum of c log2 c over the pairs with both ids != 0
  kEvXlR = 14,       // 3 limbs: sum of r' log2 r' (row sums over those pairs)
  kEvXlS = 17,       // 3 limbs: sum of s' log2 s' (column sums over those pairs)
  kEvK = 20,         // pairs with both ids != 0 and c > size_threshold (per scoring call)
  kEvStatWords = 32
};

struct EvTables {
  unsigned long long* stats;                                    // kEvStatWords
  unsigned long long *pk1, *pk2, *rkey, *ckey;                  // pair seg / gt ids, row seg id, col gt id
  uint32_t *pstate, *pcount, *rstate, *rall, *rnz, *cstate, *call, *cnz;
  unsigned long long mask;                                      // slots - 1
};

__device__ __forceinline__ unsigned long long ev_hash(unsigned long long a, unsigned long long b) {
  return rg_hash(a ^ rg_hash(b + 0x9e3779b97f4a7c15ULL));
}

// slot of key (a, b) (b ignored unless kPair), inserted if absent; -1 when no slot is found within kRgMaxProbe probes.
// *inserted = true for the one caller that created the entry.
template <bool kPair>
__device__ __forceinline__ long long ev_slot(uint32_t* state, unsigned long long* k1, unsigned long long* k2, unsigned long long a,
                                             unsigned long long b, unsigned long long mask, bool* inserted) {
  unsigned long long h = (kPair ? ev_hash(a, b) : rg_hash(a)) & mask;
  for (int probe = 0; probe < kRgMaxProbe; ++probe, h = (h + 1) & mask) {
    uint32_t st = *reinterpret_cast<volatile uint32_t*>(state + h);   // other threads insert concurrently
    if (st == 0u) {
      st = atomicCAS(&state[h], 0u, 1u);
      if (st == 0u) {                       // claimed: publish the key, then mark the slot ready
        k1[h] = a;
        if (kPair) k2[h] = b;
        __threadfence();
        atomicExch(&state[h], 2u);
        *inserted = true;
        return (long long)h;
      }
    }
    while (st == 1u) st = *reinterpret_cast<volatile uint32_t*>(state + h);   // the claimer is writing the key
    __threadfence();
    if (*reinterpret_cast<volatile unsigned long long*>(k1 + h) == a &&
        (!kPair || *reinterpret_cast<volatile unsigned long long*>(k2 + h) == b)) {
      *inserted = false;
      return (long long)h;
    }
  }
  return -1;
}

// c log2 c (0 for c < 2) added to three exact uint64 limbs: integer part, fraction bits 2^-25..2^-1 and 2^-51..2^-26
__device__ __forceinline__ void ev_xl_add(unsigned long long acc[3], uint32_t c) {
  if (c < 2u) return;
  const double t = (double)c * log2((double)c);   // >= 2: a multiple of 2^-51
  const unsigned long long ip = (unsigned long long)t;
  const unsigned long long f = (unsigned long long)((t - (double)ip) * 2251799813685248.0);   // * 2^51, exact
  acc[0] += ip;
  acc[1] += f >> 26;
  acc[2] += f & ((1ULL << 26) - 1ULL);
}

// ---- voxel pass: one run-aggregated increment per run of equal (seg, gt) pairs within a warp's 32 consecutive voxels ----
template <typename TS, typename TG>
__global__ void __launch_bounds__(kT) ev_pairs_kernel(const TS* __restrict__ seg, const TG* __restrict__ gt, int64_t n, EvTables t) {
  const int lane = ev_lane();
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / EV_WARP;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;   // voxels per sweep of the whole grid
  for (int64_t base = warp * EV_WARP; base < n; base += stride) {   // warp-uniform: every lane reaches the shuffles
    const int64_t i = base + lane;
    const bool valid = i < n;
    const unsigned long long a = valid ? (unsigned long long)seg[i] : 0ULL;
    const unsigned long long b = valid ? (unsigned long long)gt[i] : 0ULL;
    const unsigned long long pa = ev_shfl_up(a), pb = ev_shfl_up(b);
    const bool head = valid && (lane == 0 || pa != a || pb != b);
    const uint32_t ends = ev_ballot(head || !valid);           // a run ends where the next one (or the volume's end) starts
    if (!head) continue;
    const uint32_t above = ends & (uint32_t)(~0ULL << (lane + 1));
    const uint32_t run = (uint32_t)((above ? __ffs((int)above) - 1 : EV_WARP) - lane);
    bool inserted = false;
    const long long h = ev_slot<true>(t.pstate, t.pk1, t.pk2, a, b, t.mask, &inserted);
    if (h < 0) { t.stats[kEvOverflow] = 1ULL; continue; }   // table too full: the host retries with a larger one
    if (inserted) atomicAdd(&t.stats[kEvPairs], 1ULL);
    atomicAdd(&t.pcount[h], run);
  }
}

// ---- pair table -> pair statistics + row / column tables ----
__global__ void __launch_bounds__(kT) ev_margins_kernel(EvTables t) {
  unsigned long long n = 0, s1 = 0, nboth = 0, rows = 0, cols = 0, segs = 0, gts = 0, xl[3] = {0, 0, 0};
  bool overflow = false;
  const int64_t slots = (int64_t)t.mask + 1;
  // every thread runs the same number of sweeps, so that the warp sums below see all lanes
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride) {
    if (t.pstate[s] != 2u) continue;
    const unsigned long long a = t.pk1[s], b = t.pk2[s];
    const uint32_t c = t.pcount[s];
    const bool both = a != 0ULL && b != 0ULL;
    n += c;
    s1 += (unsigned long long)c * c;
    if (both) { nboth += c; ev_xl_add(xl, c); }
    bool inserted = false;
    long long h = ev_slot<false>(t.rstate, t.rkey, nullptr, a, 0ULL, t.mask, &inserted);
    if (h < 0) { overflow = true; continue; }
    if (inserted) { ++rows; segs += a != 0ULL; }
    atomicAdd(&t.rall[h], c);
    if (both) atomicAdd(&t.rnz[h], c);
    h = ev_slot<false>(t.cstate, t.ckey, nullptr, b, 0ULL, t.mask, &inserted);
    if (h < 0) { overflow = true; continue; }
    if (inserted) { ++cols; gts += b != 0ULL; }
    atomicAdd(&t.call[h], c);
    if (both) atomicAdd(&t.cnz[h], c);
  }
  const unsigned long long v[11] = {n, s1, nboth, rows, cols, segs, gts, xl[0], xl[1], xl[2], (unsigned long long)overflow};
  const int dst[11] = {kEvN, kEvS1, kEvNBoth, kEvRows, kEvCols, kEvSegIds, kEvGtIds, kEvXlC, kEvXlC + 1, kEvXlC + 2, kEvOverflow};
#pragma unroll
  for (int k = 0; k < 11; ++k) {
    const unsigned long long w = ev_warp_sum(v[k]);
    if (ev_lane() == 0 && w) atomicAdd(&t.stats[dst[k]], w);
  }
}

// ---- row / column table -> sum of squares (all voxels) and xlog2 sum (both-non-zero voxels) ----
__global__ void __launch_bounds__(kT) ev_side_kernel(const uint32_t* __restrict__ state, const uint32_t* __restrict__ all,
                                                     const uint32_t* __restrict__ nz, int64_t slots, unsigned long long* __restrict__ sq_out,
                                                     unsigned long long* __restrict__ xl_out) {
  unsigned long long sq = 0, xl[3] = {0, 0, 0};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride) {
    if (state[s] != 2u) continue;
    const unsigned long long r = all[s];
    sq += r * r;
    ev_xl_add(xl, nz[s]);
  }
  const unsigned long long v[4] = {sq, xl[0], xl[1], xl[2]};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const unsigned long long w = ev_warp_sum(v[k]);
    if (ev_lane() == 0 && w) atomicAdd(k == 0 ? sq_out : xl_out + (k - 1), w);
  }
}

// ---- edit distance: pairs with both ids != 0 that survive `r.data[r.data <= size_threshold] = 0` ----
__global__ void __launch_bounds__(kT) ev_threshold_kernel(EvTables t, double size_threshold) {
  unsigned long long k = 0;
  const int64_t slots = (int64_t)t.mask + 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride)
    if (t.pstate[s] == 2u && t.pk1[s] != 0ULL && t.pk2[s] != 0ULL && !((double)t.pcount[s] <= size_threshold)) ++k;
  k = ev_warp_sum(k);
  if (ev_lane() == 0 && k) atomicAdd(&t.stats[kEvK], k);
}
