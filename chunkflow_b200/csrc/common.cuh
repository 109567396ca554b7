// Shared declarations of the chunkflow_b200 native library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <utility>

#include "chunkflow_b200.h"

namespace cfb {

struct Int3 {
  int z, y, x;
};

inline int64_t vol(const Int3& s) { return (int64_t)s.z * s.y * s.x; }

#ifdef __CUDACC__
// max / min that are NaN when either operand is NaN, as torch's max pooling and clamp are (fmaxf / fminf return the other
// operand and would hide a broken weight from the output range check); one instruction each, like fmaxf / fminf
__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float min_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
#endif

void set_last_error(const std::string& msg);

struct CudaError : std::runtime_error {
  explicit CudaError(const std::string& m) : std::runtime_error(m) {}
};

#define CFB_CUDA(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      throw ::cfb::CudaError(std::string(#expr) + " failed: " + cudaGetErrorString(_e) +      \
                             " (" __FILE__ ":" + std::to_string(__LINE__) + ")");             \
    }                                                                                         \
  } while (0)

#define CFB_LAUNCH_CHECK() CFB_CUDA(cudaGetLastError())

#ifdef __CUDACC__
// kernel<<<grid, block, smem, stream>>>(args...), then a CudaError if the launch failed.  The host emulations under
// tests/host_emulation compile the operators with g++ and a fake runtime header that defines its own launch.
template <typename... P, typename... A>
void launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A&&... args) {
  kernel<<<grid, block, smem, stream>>>(std::forward<A>(args)...);
  CFB_LAUNCH_CHECK();
}
#endif

// The error boundary of every C-ABI entry point: an exception becomes a status code, its message cfb_last_error().
template <typename F>
int guarded(F&& f) {
  try {
    return f();
  } catch (const std::invalid_argument& ex) {
    set_last_error(ex.what());
    return CFB_ERR_INVALID_ARGUMENT;
  } catch (const CudaError& ex) {
    set_last_error(ex.what());
    return CFB_ERR_CUDA;
  } catch (const std::exception& ex) {
    set_last_error(ex.what());
    return CFB_ERR_UNSUPPORTED;
  }
}

// One device allocation, freed with its owner (on the device current at that time).
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  explicit DeviceBuffer(size_t bytes) { grow(bytes); }
  DeviceBuffer(DeviceBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    std::swap(p_, o.p_);
    std::swap(bytes_, o.bytes_);
    return *this;
  }
  ~DeviceBuffer() { reset(); }

  // Makes the buffer at least `bytes` long; a new allocation does not keep the contents.
  void grow(size_t bytes) {
    if (p_ && bytes <= bytes_) return;
    reset();
    CFB_CUDA(cudaMalloc(&p_, bytes));
    bytes_ = bytes;
  }
  void reset() {
    if (p_) cudaFree(p_);  // unchecked: also runs in destructors
    p_ = nullptr;
    bytes_ = 0;
  }
  template <typename T = void>
  T* as() const { return static_cast<T*>(p_); }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  void* p_ = nullptr;
  size_t bytes_ = 0;
};

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Patch table entry in device memory: chunk-local input start and output-buffer start.
struct PatchPos {
  int iz, iy, ix;  // input patch start inside the chunk
  int oz, oy, ox;  // start of the (cropped) output patch inside the output buffer (may be <0 / clipped)
  int flags;       // test-time augmentation variant: bit 0 transpose y<->x, bit 1 flip x, bit 2 flip y,
                   // bit 3 (kTtaChannelSym) blend the variant AND its channel-reversed copy
};

// Reference-literal --augment (transform.py:30-52,147-156): FlipLR / FlipUD act on the CHANNEL / BATCH axes of the
// 5-D buffers, so the 8 "variants" of a patch are {identity, transpose} x {as is, output channels reversed} x 2
// duplicates: two network evaluations, each blended together with its channel-reversed copy, weight 1/4.
constexpr int kTtaChannelSym = 8;

// Test-time augmentation (reference transform.py:114-145: transpose, then flip x, then flip y).
// Maps coordinates (y, x) of the TRANSFORMED patch of size (Y, X) back to the original patch.
// The same map serves the input read and, being its own inverse chain, the output write-back.
__host__ __device__ __forceinline__ void tta_map(int flags, int Y, int X, int y, int x, int& sy, int& sx) {
  const int yy = (flags & 4) ? Y - 1 - y : y;
  const int xx = (flags & 2) ? X - 1 - x : x;
  if (flags & 1) { sy = xx; sx = yy; } else { sy = yy; sx = xx; }
}

// Per-axis coverage table for the weight-volume gather: for every output coordinate the
// (ascending) list of patch axis-indices that cover it; -1 terminated.
constexpr int kMaxCover = 4;

}  // namespace cfb
