// evaluate.cu and evaluate_scores.h on the host (tests/test_evaluate_oracle.py), behind the one-lane CUDA shim of
// cuda_shim/cuda_runtime.h: every run of equal pairs has length 1.
#include <string>

#include "../../chunkflow_b200/csrc/evaluate.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }
