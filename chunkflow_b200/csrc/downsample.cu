// `downsample` on the device (DESIGN.md section 0, row f7): the reference's `downsample` command (flow/flow.py:1545-1573)
// averages uint8 images and mode-pools integer segmentations.  It calls tinybrain, a third-party package; the arithmetic
// pinned here is the reference's vendored numpy downsampler (lib/igneous/downsample.py), restated in
// oracle/downsample_oracle.py.  downsample_kernels.cuh holds the kernels and the level plan of a segmentation factor; every
// level reads its input once and writes its output once, intermediate levels going to the caller's workspace.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <stdexcept>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

#include "downsample_kernels.cuh"

DsDims ds_dims(int64_t z, int64_t y, int64_t x) {
  if (z <= 0 || y <= 0 || x <= 0) throw std::invalid_argument("downsample: bad volume size");
  return {z, y, x};
}

DsDims ds_factor(const int64_t* factor) {
  if (!factor) throw std::invalid_argument("downsample: null factor");
  return {factor[0], factor[1], factor[2]};
}

int ds_kind(int32_t dtype) {
  if (dtype == CFB_DTYPE_BOOL) return kDsBool;
  if (dtype == CFB_DTYPE_U32) return kDsU32;
  if (dtype == CFB_DTYPE_U64) return kDsU64;
  throw std::invalid_argument("downsample: a segmentation is CFB_DTYPE_U32, CFB_DTYPE_U64 or CFB_DTYPE_BOOL");
}

int64_t ds_bytes(int kind) { return kind == kDsBool ? 1 : kind == kDsU32 ? 4 : 8; }

int64_t ds_voxels(const DsDims& d) { return d.z * d.y * d.x; }

int ds_plan_or_throw(int kind, DsDims shape, DsDims factor, DsLevel* levels) {
  const char* why = "";
  const int n = ds_plan(kind, shape, factor, levels, &why);
  if (n < 0) throw std::invalid_argument(why);
  return n;
}

// bytes of the intermediate levels: every level but the last, each rounded up to 256 bytes
int64_t ds_workspace_bytes(int kind, const DsLevel* levels, int n) {
  int64_t bytes = 0;
  for (int i = 0; i + 1 < n; ++i) bytes += ceil_div64(ds_voxels(levels[i].out) * ds_bytes(kind), 256) * 256;
  return bytes;
}

void ds_check_disjoint(const void* a, int64_t a_bytes, const void* b, int64_t b_bytes) {
  const char *p = (const char*)a, *q = (const char*)b;
  if (p < q + b_bytes && q < p + a_bytes) throw std::invalid_argument("downsample: input and output overlap");
}

void ds_launch_geometry(const DsDims& o, dim3& grid, dim3& block) {
  const int64_t threads = std::min<int64_t>(256, ceil_div64(o.x, 32) * 32);
  block = dim3((unsigned)threads);
  grid = dim3((unsigned)std::min<int64_t>(ceil_div64(o.x, threads), 4096), (unsigned)std::min<int64_t>(o.y, 65535),
              (unsigned)std::min<int64_t>(o.z, 65535));
}

template <typename T>
void ds_launch_level(const DsLevel& l, int kind, const void* in, void* out, cudaStream_t s) {
  dim3 grid, block;
  ds_launch_geometry(l.out, grid, block);
  const T* src = static_cast<const T*>(in);
  T* dst = static_cast<T*>(out);
  if (l.algo == kDsStride) launch(ds_stride_kernel<T>, grid, block, 0, s, src, l.in, l.out, l.factor, dst);
  else if constexpr (sizeof(T) == 1) throw std::logic_error("downsample: a boolean volume is only strided");
  else if (l.algo == kDsCountless3d) launch(ds_countless3d_kernel<T>, grid, block, 0, s, src, l.in, l.out, dst);
  else if (kind == kDsU64) launch(ds_countless2d_kernel<T, false>, grid, block, 0, s, src, l.in, l.out, l.preserved, dst);
  else launch(ds_countless2d_kernel<T, true>, grid, block, 0, s, src, l.in, l.out, l.preserved, dst);   // widened: every id counts
}

// cfb_downsample_average_device; *vectorised, when given, is set to whether the vectorised kernel ran
int ds_average(const uint8_t* d_in, int64_t z, int64_t y, int64_t x, const int64_t factor[3], uint8_t* d_out, void* stream,
               bool* vectorised) {
  return guarded([&]() -> int {
    const DsDims s = ds_dims(z, y, x), f = ds_factor(factor);
    if (f.z <= 0 || f.y <= 0 || f.x <= 0) throw std::invalid_argument("downsample: factors below one make no sense");
    if (f.z > kDsMaxAverageBlock / f.y || f.z * f.y > kDsMaxAverageBlock / f.x)
      throw std::invalid_argument("downsample: averaging blocks of more than 65793 voxels are refused (the reference's float32 "
                                  "sum is no longer exact)");
    if (!d_in || !d_out) throw std::invalid_argument("downsample: null argument");
    const DsDims o = {ds_ceil(s.z, f.z), ds_ceil(s.y, f.y), ds_ceil(s.x, f.x)};
    ds_check_disjoint(d_in, ds_voxels(s), d_out, ds_voxels(o));
    cudaStream_t st = (cudaStream_t)stream;
    if (f.z == 1 && f.y == 1 && f.x == 1) {
      CFB_CUDA(cudaMemcpyAsync(d_out, d_in, (size_t)ds_voxels(s), cudaMemcpyDeviceToDevice, st));
      return CFB_OK;
    }
    dim3 grid, block;
    const bool vec = ds_average_vectorised(s, f, d_in, d_out);
    if (vectorised) *vectorised = vec;
    if (vec) {
      ds_launch_geometry({o.z, o.y, o.x / 8}, grid, block);
      if (f.z == 1) launch(ds_average_x2_kernel<1, 2>, grid, block, 0, st, d_in, s, o, d_out);
      else launch(ds_average_x2_kernel<2, 2>, grid, block, 0, st, d_in, s, o, d_out);
    } else {
      ds_launch_geometry(o, grid, block);
      launch(ds_average_kernel, grid, block, 0, st, d_in, s, o, f, d_out);
    }
    return CFB_OK;
  });
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int cfb_downsample_average_device(const uint8_t* d_in, int64_t z, int64_t y, int64_t x, const int64_t factor[3],
                                             uint8_t* d_out, void* stream) {
  return ds_average(d_in, z, y, x, factor, d_out, stream, nullptr);
}

extern "C" int cfb_downsample_workspace(int32_t dtype, int64_t z, int64_t y, int64_t x, const int64_t factor[3], int64_t out_zyx[3],
                                        int64_t* workspace_bytes) {
  return guarded([&]() -> int {
    const int kind = ds_kind(dtype);
    DsLevel levels[kDsMaxLevels];
    const DsDims s = ds_dims(z, y, x);
    const int n = ds_plan_or_throw(kind, s, ds_factor(factor), levels);
    const DsDims o = n ? levels[n - 1].out : s;
    if (out_zyx) { out_zyx[0] = o.z; out_zyx[1] = o.y; out_zyx[2] = o.x; }
    if (workspace_bytes) *workspace_bytes = ds_workspace_bytes(kind, levels, n);
    return CFB_OK;
  });
}

extern "C" int cfb_downsample_segmentation_device(const void* d_in, int32_t dtype, int64_t z, int64_t y, int64_t x,
                                                  const int64_t factor[3], void* d_workspace, void* d_out, void* stream) {
  return guarded([&]() -> int {
    const int kind = ds_kind(dtype);
    DsLevel levels[kDsMaxLevels];
    const DsDims s = ds_dims(z, y, x);
    const int n = ds_plan_or_throw(kind, s, ds_factor(factor), levels);
    if (!d_in || !d_out) throw std::invalid_argument("downsample: null argument");
    const int64_t esize = ds_bytes(kind);
    const int64_t work = ds_workspace_bytes(kind, levels, n);
    if (work > 0 && !d_workspace) throw std::invalid_argument("downsample: this factor needs a workspace (cfb_downsample_workspace)");
    const DsDims o = n ? levels[n - 1].out : s;
    ds_check_disjoint(d_in, ds_voxels(s) * esize, d_out, ds_voxels(o) * esize);
    if (work > 0) {
      ds_check_disjoint(d_in, ds_voxels(s) * esize, d_workspace, work);
      ds_check_disjoint(d_out, ds_voxels(o) * esize, d_workspace, work);
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
      CFB_CUDA(cudaMemcpyAsync(d_out, d_in, (size_t)(ds_voxels(s) * esize), cudaMemcpyDeviceToDevice, st));
      return CFB_OK;
    }
    const void* src = d_in;
    char* next = static_cast<char*>(d_workspace);
    for (int i = 0; i < n; ++i) {
      void* dst = i + 1 == n ? d_out : next;
      if (kind == kDsBool) ds_launch_level<uint8_t>(levels[i], kind, src, dst, st);
      else if (kind == kDsU32) ds_launch_level<uint32_t>(levels[i], kind, src, dst, st);
      else ds_launch_level<unsigned long long>(levels[i], kind, src, dst, st);
      src = dst;
      next += ceil_div64(ds_voxels(levels[i].out) * esize, 256) * 256;
    }
    return CFB_OK;
  });
}
