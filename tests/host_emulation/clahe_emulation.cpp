// clahe.cu on the host (tests/test_clahe_oracle.py), behind the one-lane CUDA shim of cuda_shim/cuda_runtime.h.
#include <string>
#include <vector>

namespace cfb {
namespace {
alignas(16) unsigned char clahe_smem[1 << 24];   // the dynamic shared memory of clahe_small_kernel
}  // namespace
}  // namespace cfb

#include "../../chunkflow_b200/csrc/clahe.cu"

namespace cfb {
static std::string last_error;
void set_last_error(const std::string& msg) { last_error = msg; }
}  // namespace cfb
extern "C" const char* cfb_last_error(void) { return cfb::last_error.c_str(); }

// One path of cfb_clahe_device forced: 0 the table path in batches of `batch` sections, 1 the small-tile path.
extern "C" int emu_clahe_path(const uint8_t* in, uint8_t* out, int64_t z, int64_t y, int64_t x, double clip, int32_t tiles_x,
                              int32_t tiles_y, int path, int64_t batch) {
  return guarded([&]() -> int {
    const ClaheGeom g = clahe_checked(z, y, x, tiles_x, tiles_y, clip);
    std::vector<uint8_t> luts(path == 1 ? 0 : (size_t)(batch * g.tiles_x * g.tiles_y * kClaheBins));
    if (path == 1) clahe_run_small(in, out, z, g, nullptr);
    else clahe_run_table(in, out, z, g, luts.data(), batch, nullptr);
    return CFB_OK;
  });
}

// The region of tiles one CTA of the small-tile path owns, and the tile size: (ry, rx, th, tw).
extern "C" void emu_small_region(int64_t y, int64_t x, int64_t tiles_x, int64_t tiles_y, int64_t* out) {
  const ClaheGeom g = clahe_geometry(y, x, tiles_x, tiles_y, 0.0);
  const ClaheRegion r = clahe_small_region(g);
  out[0] = r.ry;
  out[1] = r.rx;
  out[2] = g.th;
  out[3] = g.tw;
}
