// `gaussian-filter` and the median filter on the device (DESIGN.md section 0, row f8): the reference's
// Chunk.gaussian_filter_2d (chunk/base.py:846-853), plugins/gaussian_filter.py and plugins/median_filter.py call
// scipy.ndimage.gaussian_filter / median_filter; filter_kernels.cuh restates their arithmetic bit for bit
// (oracle/filters_oracle.py) and says how the in-place gaussian runs through a workspace of whole sections.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <stdexcept>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

#include "filter_kernels.cuh"

int64_t flt_esize(int32_t dtype) {
  if (dtype == CFB_DTYPE_U8) return 1;
  if (dtype == CFB_DTYPE_F32) return 4;
  throw std::invalid_argument("filters: the chunk is CFB_DTYPE_U8 or CFB_DTYPE_F32");
}

FltDims flt_dims(int64_t c, int64_t z, int64_t y, int64_t x) {
  if (c <= 0 || z <= 0 || y <= 0 || x <= 0) throw std::invalid_argument("filters: bad chunk size");
  return {{c, z, y, x}};
}

// sections per batch: as many as fit kFltWorkspaceTarget, at least one, at most all
int64_t flt_batch(const FltDims& d, int64_t esize) {
  const int64_t section = d.n[0] * d.n[2] * d.n[3] * esize;
  return std::max<int64_t>(1, std::min<int64_t>(d.n[1], kFltWorkspaceTarget / section));
}

FltWeights flt_weights(const double* w, int32_t r, const char* axis) {
  FltWeights out{};
  if (!w) {
    if (r != 0) throw std::invalid_argument(std::string("gaussian filter: null weights for axis ") + axis);
    out.w[0] = 1.0;   // no pass: x * 1 cast back is x
    return out;
  }
  if (r < 0 || r > kFltMaxRadius) throw std::invalid_argument("gaussian filter: the radius is 0 .. 64");
  std::memcpy(out.w, w, sizeof(double) * (r + 1));
  out.r = r;
  return out;
}

dim3 flt_grid_1d(int64_t work) { return dim3((unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(work, kFltThreads), 8192))); }

template <typename T>
void flt_launch_yx(const T* src, FltPlanes sp, T* dst, FltPlanes dp, int64_t nc, int64_t nz, int64_t Y, int64_t X,
                   const FltWeights& wy, const FltWeights& wx, cudaStream_t st) {
  const int64_t smem = flt_yx_smem_bytes(wy.r, wx.r, sizeof(T));
  CFB_CUDA(cudaFuncSetAttribute(flt_gaussian_yx_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)std::min<int64_t>(ceil_div64(X, kFltTx), 65535), (unsigned)std::min<int64_t>(ceil_div64(Y, kFltTy), 65535),
                  (unsigned)std::min<int64_t>(nc * nz, 65535));
  launch(flt_gaussian_yx_kernel<T>, grid, kFltThreads, smem, st, src, sp, dst, dp, nc, nz, Y, X, wy, wx);
}

// in place, in batches of `batch` sections through `work`
template <typename T>
void flt_gaussian(T* data, const FltDims& d, const FltWeights& wc, bool channel_pass, const FltWeights& wy,
                  const FltWeights& wx, T* work, int64_t batch, cudaStream_t st) {
  const int64_t C = d.n[0], Z = d.n[1], Y = d.n[2], X = d.n[3], yx = Y * X;
  for (int64_t z0 = 0; z0 < Z; z0 += batch) {
    const int64_t nb = std::min(batch, Z - z0);
    const FltPlanes chunk{Z * yx, yx}, ws{nb * yx, yx};
    T* at = data + z0 * yx;
    if (channel_pass) {
      const dim3 grid((unsigned)std::min<int64_t>(ceil_div64(yx, kFltThreads), 4096), (unsigned)std::min<int64_t>(nb, 65535),
                      (unsigned)std::min<int64_t>(C, 65535));
      launch(flt_gaussian_c_kernel<T>, grid, kFltThreads, 0, st, at, chunk, work, ws, C, nb, yx, wc);
      flt_launch_yx<T>(work, ws, at, chunk, C, nb, Y, X, wy, wx, st);
    } else {
      flt_launch_yx<T>(at, chunk, work, ws, C, nb, Y, X, wy, wx, st);
      for (int64_t c = 0; c < C; ++c)
        CFB_CUDA(cudaMemcpyAsync(at + c * Z * yx, work + c * nb * yx, (size_t)(nb * yx * sizeof(T)), cudaMemcpyDeviceToDevice, st));
    }
  }
}

template <typename T>
void flt_launch_median(const T* in, const FltDims& n, const FltDims& size, int mode, T* out, cudaStream_t st) {
  const int path = flt_median_path(size);
  if (path < 0) {
    launch(flt_median_z3_kernel<T>, flt_grid_1d(n.n[0] * n.n[2] * n.n[3]), kFltThreads, 0, st, in, n, mode, out);
  } else {
    const dim3 grid = flt_grid_1d(n.n[0] * n.n[1] * n.n[2] * n.n[3]);
    if (path == 4) launch(flt_median_kernel<T, 4>, grid, kFltThreads, 0, st, in, n, size, mode, out);
    else if (path == 16) launch(flt_median_kernel<T, 16>, grid, kFltThreads, 0, st, in, n, size, mode, out);
    else if (path == 32) launch(flt_median_kernel<T, 32>, grid, kFltThreads, 0, st, in, n, size, mode, out);
    else launch(flt_median_kernel<T, 0>, grid, kFltThreads, 0, st, in, n, size, mode, out);
  }
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_gaussian_filter_workspace(int32_t dtype, int64_t c, int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    const int64_t esize = flt_esize(dtype);
    const FltDims d = flt_dims(c, z, y, x);
    if (!workspace_bytes) throw std::invalid_argument("gaussian filter: null argument");
    *workspace_bytes = flt_batch(d, esize) * c * y * x * esize;
    return CFB_OK;
  });
}

extern "C" int cfb_gaussian_filter_device(void* d_data, int32_t dtype, int64_t c, int64_t z, int64_t y, int64_t x,
                                          const double* w_c, int32_t r_c, const double* w_y, int32_t r_y, const double* w_x,
                                          int32_t r_x, void* d_workspace, int64_t workspace_bytes, void* stream) {
  return guarded([&]() -> int {
    const int64_t esize = flt_esize(dtype);
    const FltDims d = flt_dims(c, z, y, x);
    const FltWeights wc = flt_weights(w_c, r_c, "c"), wy = flt_weights(w_y, r_y, "y"), wx = flt_weights(w_x, r_x, "x");
    if (!d_data || !d_workspace) throw std::invalid_argument("gaussian filter: null argument");
    const int64_t batch = flt_batch(d, esize), need = batch * c * y * x * esize;
    if (workspace_bytes < need) throw std::invalid_argument("gaussian filter: the workspace is smaller than cfb_gaussian_filter_workspace");
    const char *p = (const char*)d_data, *q = (const char*)d_workspace;
    if (p < q + need && q < p + c * z * y * x * esize) throw std::invalid_argument("gaussian filter: chunk and workspace overlap");
    cudaStream_t st = (cudaStream_t)stream;
    if (!w_c && !w_y && !w_x) return CFB_OK;
    if (dtype == CFB_DTYPE_U8)
      flt_gaussian<uint8_t>((uint8_t*)d_data, d, wc, w_c != nullptr, wy, wx, (uint8_t*)d_workspace, batch, st);
    else
      flt_gaussian<float>((float*)d_data, d, wc, w_c != nullptr, wy, wx, (float*)d_workspace, batch, st);
    return CFB_OK;
  });
}

extern "C" int cfb_median_filter_device(const void* d_in, int32_t dtype, int64_t c, int64_t z, int64_t y, int64_t x,
                                        const int64_t size[4], int32_t mode, void* d_out, void* stream) {
  return guarded([&]() -> int {
    const int64_t esize = flt_esize(dtype);
    const FltDims n = flt_dims(c, z, y, x);
    if (!size) throw std::invalid_argument("median filter: null size");
    const FltDims s = {{size[0], size[1], size[2], size[3]}};
    int64_t volume = 1;
    for (int d = 0; d < 4; ++d) {
      if (s.n[d] < 1 || s.n[d] > kFltMaxWindow) throw std::invalid_argument("median filter: every window extent is 1 .. 125");
      volume *= s.n[d];
    }
    if (volume > kFltMaxWindow) throw std::invalid_argument("median filter: windows of more than 125 elements (5x5x5) are refused");
    if (mode < kFltReflect || mode > kFltConstant) throw std::invalid_argument("median filter: unknown mode");
    if (!d_in || !d_out) throw std::invalid_argument("median filter: null argument");
    const int64_t bytes = c * z * y * x * esize;
    const char *p = (const char*)d_in, *q = (const char*)d_out;
    if (p < q + bytes && q < p + bytes) throw std::invalid_argument("median filter: input and output overlap");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == CFB_DTYPE_U8) flt_launch_median<uint8_t>((const uint8_t*)d_in, n, s, mode, (uint8_t*)d_out, st);
    else flt_launch_median<float>((const float*)d_in, n, s, mode, (float*)d_out, st);
    return CFB_OK;
  });
}
