// downsample.cu on the host (tests/test_downsample_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h.
#include <string>

#include "../../chunkflow_b200/csrc/downsample.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }

// cfb_downsample_average_device -> 1 when the vectorised kernel ran, 0 for the generic one, or the error code.
extern "C" int emu_average(const uint8_t* in, int64_t z, int64_t y, int64_t x, const int64_t* factor, uint8_t* out) {
  bool vectorised = false;
  const int rc = ds_average(in, z, y, x, factor, out, nullptr, &vectorised);
  return rc != CFB_OK ? rc : vectorised ? 1 : 0;
}

// The level plan: -> levels (-1 when refused); plan[5 i ..] = algorithm, preserved axis, output z, y, x of level i.
extern "C" int emu_plan(int kind, int64_t z, int64_t y, int64_t x, int64_t fz, int64_t fy, int64_t fx, int64_t* plan) {
  DsLevel levels[kDsMaxLevels];
  const char* why = "";
  const int n = ds_plan(kind, DsDims{z, y, x}, DsDims{fz, fy, fx}, levels, &why);
  for (int i = 0; i < n; ++i) {
    const int64_t row[5] = {levels[i].algo, levels[i].preserved, levels[i].out.z, levels[i].out.y, levels[i].out.x};
    std::memcpy(plan + 5 * i, row, sizeof(row));
  }
  return n;
}
