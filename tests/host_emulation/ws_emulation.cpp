// segmentation.cu on the host (tests/test_segmentation_agglomerate.py), behind the one-lane CUDA shim of
// cuda_shim/cuda_runtime.h.  The ranking of the union-find roots in raster order is three kernels whose threads cooperate
// through shared memory; launching one of them runs what it computes serially instead (defined below the library).
#include <string>

#include "scan_blocks.h"

template <typename... A>
void launch(void (*kernel)(const uint32_t*, uint32_t*, int64_t, uint32_t*), dim3, dim3, size_t, cudaStream_t, A&&... args);
template <typename... A>
void launch(void (*kernel)(const uint32_t*, const uint32_t*, int64_t, const uint32_t*, uint32_t*), dim3, dim3, size_t, cudaStream_t,
            A&&... args);

#include "../../chunkflow_b200/csrc/segmentation.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }

// cc_flatten_count_kernel: every foreground voxel pointed at its root, the roots of every scan block counted
template <typename... A>
void launch(void (*kernel)(const uint32_t*, uint32_t*, int64_t, uint32_t*), dim3, dim3, size_t, cudaStream_t, A&&... args) {
  if (kernel != cc_flatten_count_kernel) return kernel(args...);
  [](const uint32_t* val, uint32_t* P, int64_t n, uint32_t* block_count) {
    for (int64_t i = 0; i < n; ++i) {
      if (i % kScanBlock == 0) block_count[i / kScanBlock] = 0;
      if (val[i] && (P[i] = uf_find(P, (uint32_t)i)) == (uint32_t)i) ++block_count[i / kScanBlock];
    }
  }(args...);
}

// cc_rank_kernel: the rank of every root, its block's base plus the roots before it in the block
template <typename... A>
void launch(void (*kernel)(const uint32_t*, const uint32_t*, int64_t, const uint32_t*, uint32_t*), dim3, dim3, size_t, cudaStream_t,
            A&&... args) {
  if (kernel != cc_rank_kernel) return kernel(args...);
  [](const uint32_t* val, const uint32_t* P, int64_t n, const uint32_t* block_base, uint32_t* rank) {
    uint32_t next = 0;
    for (int64_t i = 0; i < n; ++i) {
      if (i % kScanBlock == 0) next = block_base[i / kScanBlock];
      if (val[i] && P[i] == (uint32_t)i) rank[i] = next++;
    }
  }(args...);
}
