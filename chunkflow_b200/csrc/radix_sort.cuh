// Stable LSD radix sort of (uint64 id, uint64 value) pairs by the low bits of the id, and the chunked exclusive scan of uint32
// it is built on.  Written for `mesh` (sorting its streams by object) and shared with `skeletonize` (sorting the voxels of
// every object by geodesic distance).  The histograms are digit-major, one column per chunk of kMcChunk items, so that their
// exclusive scan is the stable scatter's base; one thread owns a chunk, which is also how the one-lane host emulation runs it.
// NOT a stand-alone header: included inside the library's anonymous namespace, after `kMcThreads` (threads per block) and
// raster_scan.cuh (cc_scan_blocks_kernel: the scan of the chunk sums).
#pragma once

constexpr int kMcChunk = 1024;   // items per thread in the scans and the radix sort

int64_t mc_chunks(int64_t items) { return ceil_div64(items, kMcChunk); }
int mc_grid_size(int64_t work) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(work, kMcThreads), 132 * 8)); }

// ---- exclusive scan of n uint32 in chunks of kMcChunk: chunk sums, their scan (cc_scan_blocks_kernel), chunk scans ----
__global__ void __launch_bounds__(kMcThreads) mc_chunk_sum_kernel(const uint32_t* __restrict__ a, int64_t n, uint32_t* __restrict__ sums) {
  const int64_t chunks = (n + kMcChunk - 1) / kMcChunk, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chunks; c += stride) {
    uint32_t s = 0;
    for (int64_t i = c * kMcChunk; i < n && i < (c + 1) * kMcChunk; ++i) s += a[i];
    sums[c] = s;
  }
}

__global__ void __launch_bounds__(kMcThreads) mc_chunk_scan_kernel(uint32_t* __restrict__ a, int64_t n, const uint32_t* __restrict__ base) {
  const int64_t chunks = (n + kMcChunk - 1) / kMcChunk, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chunks; c += stride) {
    uint32_t s = base[c];
    for (int64_t i = c * kMcChunk; i < n && i < (c + 1) * kMcChunk; ++i) {
      const uint32_t v = a[i];
      a[i] = s;
      s += v;
    }
  }
}

// ---- one 8-bit digit of the stable radix sort by id ----
__global__ void __launch_bounds__(kMcThreads) mc_radix_hist_kernel(const unsigned long long* __restrict__ ids, int64_t n, int shift,
                                                                    uint32_t* __restrict__ hist) {   // hist[digit * chunks + chunk]
  const int64_t chunks = (n + kMcChunk - 1) / kMcChunk, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chunks; c += stride) {
    uint32_t h[256];
    for (int d = 0; d < 256; ++d) h[d] = 0;
    for (int64_t i = c * kMcChunk; i < n && i < (c + 1) * kMcChunk; ++i) ++h[(ids[i] >> shift) & 255u];
    for (int d = 0; d < 256; ++d) hist[d * chunks + c] = h[d];
  }
}

__global__ void __launch_bounds__(kMcThreads) mc_radix_scatter_kernel(const unsigned long long* __restrict__ ids,
                                                                       const unsigned long long* __restrict__ vals, int64_t n, int shift,
                                                                       const uint32_t* __restrict__ base, unsigned long long* __restrict__ ids_out,
                                                                       unsigned long long* __restrict__ vals_out) {
  const int64_t chunks = (n + kMcChunk - 1) / kMcChunk, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chunks; c += stride) {
    uint32_t h[256];
    for (int d = 0; d < 256; ++d) h[d] = base[d * chunks + c];
    for (int64_t i = c * kMcChunk; i < n && i < (c + 1) * kMcChunk; ++i) {
      const uint32_t j = h[(ids[i] >> shift) & 255u]++;
      ids_out[j] = ids[i];
      vals_out[j] = vals[i];
    }
  }
}

// exclusive scan of n uint32 in place -> the total
uint32_t mc_scan(uint32_t* a, int64_t n, uint32_t* sums, cudaStream_t s) {
  const int64_t chunks = mc_chunks(n);
  launch(mc_chunk_sum_kernel, mc_grid_size(chunks), kMcThreads, 0, s, a, n, sums);
  launch(cc_scan_blocks_kernel, 1, 1024, 0, s, sums, chunks, sums + chunks);
  launch(mc_chunk_scan_kernel, mc_grid_size(chunks), kMcThreads, 0, s, a, n, (const uint32_t*)sums);
  uint32_t total = 0;
  CFB_CUDA(cudaMemcpyAsync(&total, sums + chunks, 4, cudaMemcpyDeviceToHost, s));
  CFB_CUDA(cudaStreamSynchronize(s));
  return total;
}

// stable sort of (ids, vals) by the low `bits` bits of the ids; the result is back in ids, vals (an even number of passes)
void mc_sort(unsigned long long* ids, unsigned long long* vals, unsigned long long* ids2, unsigned long long* vals2, int64_t n, int bits,
             uint32_t* hist, uint32_t* sums, cudaStream_t s) {
  const int64_t chunks = mc_chunks(n);
  for (int shift = 0; shift < bits; shift += 8) {
    launch(mc_radix_hist_kernel, mc_grid_size(chunks), kMcThreads, 0, s, (const unsigned long long*)ids, n, shift, hist);
    mc_scan(hist, 256 * chunks, sums, s);
    launch(mc_radix_scatter_kernel, mc_grid_size(chunks), kMcThreads, 0, s, (const unsigned long long*)ids,
           (const unsigned long long*)vals, n, shift, (const uint32_t*)hist, ids2, vals2);
    std::swap(ids, ids2);
    std::swap(vals, vals2);
  }
}

