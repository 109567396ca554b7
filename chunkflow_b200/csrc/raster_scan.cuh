// Second level of the two-level raster-order ranking that numbers objects 1..N by their first voxel: shared by
// `connected-components` / the watershed (segmentation.cu: roots of the union-find) and `remap` (relabel.cu: first voxels of
// the surviving labels).  The first level (flags per block of consecutive voxels -> one count per block) and the third (rank
// inside the block + the block's base) belong to the caller, which knows where its flags live.
// NOT a stand-alone header: included inside the library's anonymous namespace.
#pragma once

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
