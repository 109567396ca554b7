// `clahe` on the device (DESIGN.md section 0, row f9): the reference's plugins/clahe.py runs
// cv2.createCLAHE(clipLimit, tileGridSize).apply on every z section of a uint8 image; clahe_kernels.cuh restates OpenCV's
// arithmetic bit for bit (oracle/clahe_oracle.py) and describes the two paths and the workspace of tile LUTs.
#include <algorithm>
#include <cstdint>
#include <stdexcept>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

#include "clahe_kernels.cuh"

ClaheGeom clahe_checked(int64_t z, int64_t y, int64_t x, int32_t tiles_x, int32_t tiles_y, double clip_limit) {
  if (z <= 0 || y <= 0 || x <= 0) throw std::invalid_argument("clahe: bad chunk size");
  if (tiles_x < 1 || tiles_y < 1) throw std::invalid_argument("clahe: the tile grid has at least one tile along each axis");
  if (y > kClaheMaxSide || x > kClaheMaxSide) throw std::invalid_argument("clahe: a section side is at most 2^24 pixels");
  const ClaheGeom g = clahe_geometry(y, x, tiles_x, tiles_y, clip_limit);
  if (g.th * g.tiles_y * g.tw * g.tiles_x > INT32_MAX)
    throw std::invalid_argument("clahe: a padded section is at most 2^31 - 1 pixels (OpenCV's int sizes)");
  return g;
}

// sections per batch of the table path: as many as have their LUTs fit kClaheWorkspaceTarget, at least one, at most all;
// the small-tile path needs no workspace
int64_t clahe_batch(const ClaheGeom& g, int64_t z) {
  const int64_t per_section = g.tiles_x * g.tiles_y * kClaheBins;
  return std::max<int64_t>(1, std::min<int64_t>(z, kClaheWorkspaceTarget / per_section));
}

int64_t clahe_workspace_bytes(const ClaheGeom& g, int64_t z) {
  return clahe_small_tiles(g) ? 0 : clahe_batch(g, z) * g.tiles_x * g.tiles_y * kClaheBins;
}

void clahe_run_small(const uint8_t* in, uint8_t* out, int64_t z, const ClaheGeom& g, cudaStream_t st) {
  const ClaheRegion reg = clahe_small_region(g);
  const int64_t regions = ceil_div64(g.tiles_x, reg.rx) * ceil_div64(g.tiles_y, reg.ry);
  const int smem = (int)clahe_small_smem_bytes(g, reg);
  CFB_CUDA(cudaFuncSetAttribute(clahe_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const dim3 grid((unsigned)std::min<int64_t>(regions, 1 << 20), (unsigned)std::min<int64_t>(z, 65535));
  launch(clahe_small_kernel, grid, kClaheThreads, smem, st, in, out, z, g, reg);
}

// the table path in batches of `batch` sections, whose LUTs fill `luts`
void clahe_run_table(const uint8_t* in, uint8_t* out, int64_t z, const ClaheGeom& g, uint8_t* luts, int64_t batch, cudaStream_t st) {
  const int64_t section = g.H * g.W, tiles = g.tiles_x * g.tiles_y;
  for (int64_t z0 = 0; z0 < z; z0 += batch) {
    const int64_t nb = std::min(batch, z - z0);
    const dim3 grid((unsigned)std::min<int64_t>(tiles, 1 << 20), (unsigned)std::min<int64_t>(nb, 65535));
    launch(clahe_lut_kernel, grid, kClaheThreads, 0, st, in + z0 * section, nb, g, luts);
    launch(clahe_table_kernel, grid, kClaheThreads, 0, st, in + z0 * section, out + z0 * section, nb, g, luts);
  }
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_clahe_workspace(int64_t z, int64_t y, int64_t x, int32_t tiles_x, int32_t tiles_y, int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    const ClaheGeom g = clahe_checked(z, y, x, tiles_x, tiles_y, 0.0);
    if (!workspace_bytes) throw std::invalid_argument("clahe: null argument");
    *workspace_bytes = clahe_workspace_bytes(g, z);
    return CFB_OK;
  });
}

extern "C" int cfb_clahe_device(const void* d_in, void* d_out, int64_t z, int64_t y, int64_t x, double clip_limit, int32_t tiles_x,
                                int32_t tiles_y, void* d_workspace, int64_t workspace_bytes, void* stream) {
  return guarded([&]() -> int {
    const ClaheGeom g = clahe_checked(z, y, x, tiles_x, tiles_y, clip_limit);
    if (!d_in || !d_out) throw std::invalid_argument("clahe: null argument");
    const int64_t bytes = z * y * x, need = clahe_workspace_bytes(g, z);
    const char *p = (const char*)d_in, *q = (const char*)d_out, *w = (const char*)d_workspace;
    if (p < q + bytes && q < p + bytes) throw std::invalid_argument("clahe: input and output overlap");
    if (need > 0) {
      if (!d_workspace) throw std::invalid_argument("clahe: null workspace");
      if (workspace_bytes < need) throw std::invalid_argument("clahe: the workspace is smaller than cfb_clahe_workspace");
      if ((w < p + bytes && p < w + need) || (w < q + bytes && q < w + need))
        throw std::invalid_argument("clahe: the workspace overlaps the input or the output");
    }
    if (clahe_small_tiles(g))
      clahe_run_small((const uint8_t*)d_in, (uint8_t*)d_out, z, g, (cudaStream_t)stream);
    else
      clahe_run_table((const uint8_t*)d_in, (uint8_t*)d_out, z, g, (uint8_t*)d_workspace, clahe_batch(g, z), (cudaStream_t)stream);
    return CFB_OK;
  });
}
