// One index map per boundary mode, shared by the smoothing filters (filter_kernels.cuh, DESIGN.md section 0, row f8) and
// `clahe` (clahe_kernels.cuh, row f9).  Included inside the anonymous namespace of each .cu file.
#pragma once

enum FltMode { kFltReflect = 0, kFltNearest = 1, kFltMirror = 2, kFltWrap = 3, kFltConstant = 4 };

// Index i of a line of n elements -> 0..n-1, or -1 where the constant mode reads its 0.
__device__ __forceinline__ int64_t flt_fold(int64_t i, int64_t n, int mode) {
  if (i >= 0 && i < n) return i;
  switch (mode) {
    case kFltReflect: {   // d c b a | a b c d | d c b a (period 2n)
      int64_t k = i % (2 * n);
      if (k < 0) k += 2 * n;
      return k >= n ? 2 * n - 1 - k : k;
    }
    case kFltNearest: return i < 0 ? 0 : n - 1;
    case kFltMirror: {    // d c b | a b c d | c b a (period 2n - 2); one element mirrors onto itself
      if (n == 1) return 0;
      int64_t k = i % (2 * n - 2);
      if (k < 0) k += 2 * n - 2;
      return k >= n ? 2 * n - 2 - k : k;
    }
    case kFltWrap: {
      int64_t k = i % n;
      return k < 0 ? k + n : k;
    }
    default: return -1;
  }
}
