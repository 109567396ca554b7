// Open-addressing tables whose keys may be ANY uint64 (0 and 2^64 - 1 included), shared by the contingency table
// (evaluate_kernels.cuh) and the label table (label_table.cuh).  No key value can mark an empty slot, so each slot carries a
// state word (0 empty, 1 being written, 2 ready) and the keys are written by the thread that claimed the slot.  Also the
// warp helpers both use to combine runs of equal keys before the atomics.
// NOT a stand-alone header: included inside the library's anonymous namespace; the CUDA shim of the host emulations
// (tests/host_emulation/cuda_shim) defines EV_WARP = 1 and the ev_* helpers for a one-lane warp first.
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
