// cc_scan_blocks_kernel (raster_scan.cuh) is one block of 1024 threads that scan together, which one lane cannot stand in
// for: launching it runs the same exclusive scan of the block counts serially.  Included before relabel.cu or segmentation.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace cfb {
namespace {
void cc_scan_blocks_kernel(uint32_t* block_count, int64_t nblocks, uint32_t* num_labels);
}  // namespace
}  // namespace cfb

template <typename... A>
void launch(void (*kernel)(uint32_t*, int64_t, uint32_t*), dim3, dim3, size_t, cudaStream_t, A&&... args) {
  if (kernel != cfb::cc_scan_blocks_kernel) return kernel(args...);
  [](uint32_t* block_count, int64_t nblocks, uint32_t* num_labels) {
    uint32_t total = 0;
    for (int64_t i = 0; i < nblocks; ++i) total += std::exchange(block_count[i], total);
    *num_labels = total;
  }(args...);
}
