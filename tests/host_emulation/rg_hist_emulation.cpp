// The histogram region graph of segmentation.cu on the host (tests/test_agglomerate_quantile.py), behind the one-lane CUDA
// shim of cuda_shim/cuda_runtime.h: both passes over the faces, the two compactions and the host side of the read.  The
// fragments come from the tests (the watershed is covered by ws_emulation.cpp).
#include <string>

#include "../../chunkflow_b200/csrc/segmentation.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }
