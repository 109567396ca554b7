// skeleton.cu on the host (tests/test_skeleton_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h: one
// thread walks every row, column, tile, object and path voxel, so every kernel's stride loops cover the whole volume.
#include <string>

#include "scan_blocks.h"
#include "../../chunkflow_b200/csrc/skeleton.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }
