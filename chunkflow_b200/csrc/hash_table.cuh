// Open-addressing hash tables in global memory, shared by the region graph (watershed_kernels.cuh) and the contingency
// table (evaluate_kernels.cuh).  Linear probing from rg_hash(key) & mask; a key that finds no place within kRgMaxProbe
// slots raises the table's overflow flag and the host retries with a larger table (CFB_ERR_CAPACITY).
// NOT a stand-alone header: included inside the library's anonymous namespace.
#pragma once

constexpr int kRgMaxProbe = 1024;

// the 64-bit finaliser of MurmurHash3
__device__ __forceinline__ unsigned long long rg_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
}
