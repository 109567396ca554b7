// A fake CUDA runtime for the host emulations (tests/host_emulation/*_emulation.cpp).  They compile an operator's .cu with
// g++ and `-I tests/host_emulation/cuda_shim`, so common.cuh includes this header instead of the real one.  Device memory is
// host memory and the stream calls are synchronous.  launch() runs a kernel once, as one thread in a grid and a block of
// 1 x 1 x 1: every grid-stride loop walks all the work, a warp has one lane (EV_WARP 1) and an atomic is a plain
// read-modify-write.  Kernels whose threads cooperate through shared memory cannot run that way (see the emulations).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <utility>

#define __global__
#define __device__
#define __host__
#define __constant__
#define __shared__
#define __forceinline__ inline
#define __restrict__
#define __align__(n) __attribute__((aligned(n)))
#define __launch_bounds__(...)

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
static const dim3 blockIdx(0, 0, 0), threadIdx(0, 0, 0), blockDim, gridDim;

struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }

template <typename T> struct EmuSame { typedef T type; };   // the operand takes the type of the address
template <typename T> T atomicAdd(T* p, typename EmuSame<T>::type v) { const T o = *p; *p = o + v; return o; }
template <typename T> T atomicMin(T* p, typename EmuSame<T>::type v) { const T o = *p; if (v < o) *p = v; return o; }
template <typename T> T atomicMax(T* p, typename EmuSame<T>::type v) { const T o = *p; if (o < v) *p = v; return o; }
template <typename T> T atomicOr(T* p, typename EmuSame<T>::type v) { const T o = *p; *p = o | v; return o; }
template <typename T> T atomicExch(T* p, typename EmuSame<T>::type v) { const T o = *p; *p = v; return o; }
template <typename T> T atomicCAS(T* p, typename EmuSame<T>::type cmp, typename EmuSame<T>::type v) {
  const T o = *p;
  if (o == cmp) *p = v;
  return o;
}
using std::max;   // the CUDA headers' min and max
using std::min;
inline void __syncthreads() {}
inline void __threadfence() {}
template <typename T> T __ldg(const T* p) { return *p; }
template <typename T> T __shfl_sync(unsigned, T v, int) { return v; }   // one lane: every lane read is the lane itself
template <typename T> T __shfl_up_sync(unsigned, T v, unsigned) { return v; }
template <typename T> T __shfl_xor_sync(unsigned, T v, int) { return v; }
inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
inline int __ffs(int v) { return __builtin_ffs(v); }

// Every operation rounded on its own: the emulations build with -ffp-contract=off, so a * b + c is not fused either.
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline int __float2int_rn(float a) { return (int)std::nearbyint(a); }   // the default rounding mode: half to even
inline long long __double2ll_rn(double a) { return std::llrint(a); }
inline unsigned __double2uint_rz(double a) { return (unsigned)a; }
inline float __double2float_rn(double a) { return (float)a; }
inline float __int_as_float(int v) { float f; std::memcpy(&f, &v, sizeof f); return f; }

// the warp helpers of state_table.cuh for a one-lane warp
#define EV_WARP 1
inline int ev_lane() { return 0; }
inline unsigned long long ev_shfl_up(unsigned long long v) { return v; }
inline uint32_t ev_ballot(bool p) { return p ? 1u : 0u; }
inline unsigned long long ev_warp_sum(unsigned long long v) { return v; }

enum cudaError_t { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
typedef struct CUstream_st* cudaStream_t;

inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "out of memory"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaMalloc(void** p, size_t bytes) { *p = std::malloc(bytes); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t bytes, cudaStream_t = nullptr) { std::memset(p, v, bytes); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind, cudaStream_t = nullptr) {
  std::memcpy(dst, src, bytes);
  return cudaSuccess;
}
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
template <typename F> cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

// common.cuh's launch on the host: one call of the kernel, whatever the grid, the block and the shared memory
template <typename... P, typename... A>
void launch(void (*kernel)(P...), dim3, dim3, size_t, cudaStream_t, A&&... args) {
  kernel(std::forward<A>(args)...);
}
