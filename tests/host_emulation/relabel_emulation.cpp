// relabel.cu on the host (tests/test_relabel_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h: a
// "warp" holds the 2, 4 or 16 ids of one 16-byte load, so runs are combined inside a lane but never across lanes.
#include <string>

#include "scan_blocks.h"
#include "../../chunkflow_b200/csrc/relabel.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }
