// fill_holes.cu on the host (tests/test_fill_holes_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h: one
// thread walks every voxel, face voxel and table slot; a "warp" has one lane, so every pair is inserted on its own.
#include <string>

#include "scan_blocks.h"
#include "../../chunkflow_b200/csrc/fill_holes.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }
