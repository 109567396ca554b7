// mesh.cu on the host (tests/test_mesh_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h: one thread
// walks every block of cubes, so the block scans of the count and emit passes are serial.
#include <string>

#include "scan_blocks.h"
#include "../../chunkflow_b200/csrc/mesh.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }
