// filters.cu on the host (tests/test_filters_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h.
#include <string>
#include <vector>

namespace cfb {
namespace {
alignas(16) unsigned char flt_smem[1 << 20];   // the dynamic shared memory of flt_gaussian_yx_kernel
}  // namespace
}  // namespace cfb

#include "../../chunkflow_b200/csrc/filters.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }

// cfb_gaussian_filter_device with batches of `batch` sections (the library's choice is flt_batch).
extern "C" int emu_gaussian(int32_t dtype, void* data, int64_t c, int64_t z, int64_t y, int64_t x, const double* w_c, int32_t r_c,
                            const double* w_y, int32_t r_y, const double* w_x, int32_t r_x, int64_t batch) {
  return guarded([&]() -> int {
    const FltDims d = flt_dims(c, z, y, x);
    const FltWeights wc = flt_weights(w_c, r_c, "c"), wy = flt_weights(w_y, r_y, "y"), wx = flt_weights(w_x, r_x, "x");
    std::vector<char> work((size_t)(batch * c * y * x * flt_esize(dtype)));
    if (dtype == CFB_DTYPE_U8) flt_gaussian<uint8_t>((uint8_t*)data, d, wc, w_c != nullptr, wy, wx, (uint8_t*)work.data(), batch, nullptr);
    else flt_gaussian<float>((float*)data, d, wc, w_c != nullptr, wy, wx, (float*)work.data(), batch, nullptr);
    return CFB_OK;
  });
}

// The median kernel cfb_median_filter_device runs for a window of `size`: -1 the z walk, else the register capacity, 0 the
// local-array kernel.
extern "C" int emu_median_path(const int64_t* size) { return flt_median_path(FltDims{{size[0], size[1], size[2], size[3]}}); }
