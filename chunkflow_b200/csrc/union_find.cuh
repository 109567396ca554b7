// Label-equivalence union-find over the voxels' linear indices (lock-free: a root search and an atomicMin on the larger root),
// shared by `connected-components` and the watershed (segmentation.cu), by `skeletonize` (skeleton.cu, 26-connected objects
// of uint32 or uint64 ids) and by `fill-segmentation-holes` (fill_holes.cu, 6-connected components of every value, 0
// included, or of the background alone).  The root of a set is its smallest index.
// NOT a stand-alone header: included inside the library's anonymous namespace (after `Int3`).
#pragma once

__device__ __forceinline__ uint32_t uf_find(const uint32_t* P, uint32_t x) {
  uint32_t p = P[x];
  while (p != x) { x = p; p = P[x]; }
  return x;
}

__device__ __forceinline__ void uf_unite(uint32_t* P, uint32_t a, uint32_t b) {
  bool done = false;
  do {
    a = uf_find(P, a);
    b = uf_find(P, b);
    if (a < b) {
      const uint32_t old = atomicMin(&P[b], a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const uint32_t old = atomicMin(&P[a], b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

// backward half of the 26-neighbourhood, ordered so that the first 3 are the face neighbours (6-connectivity), the first 9
// the face + edge neighbours (18) and all 13 the full neighbourhood (26)
__constant__ int kNb[13][3] = {{0, 0, -1}, {0, -1, 0}, {-1, 0, 0},
                               {0, -1, -1}, {0, -1, 1}, {-1, 0, -1}, {-1, 0, 1}, {-1, -1, 0}, {-1, 1, 0},
                               {-1, -1, -1}, {-1, -1, 1}, {-1, 1, -1}, {-1, 1, 1}};

// which voxels join their equal neighbours: the non-zero ones, every one, or the zero ones (for float32, +0 and -0 are zero
// and NaN is not)
enum { kJoinNonZero = 0, kJoinAll = 1, kJoinZero = 2 };

template <typename V, int kJoin = kJoinNonZero>
__global__ void __launch_bounds__(256) cc_merge_kernel(const V* __restrict__ val, uint32_t* __restrict__ P, Int3 sz, int nnb) {
  const int64_t n = (int64_t)sz.z * sz.y * sz.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const V v = val[i];
    if (kJoin == kJoinNonZero ? !v : kJoin == kJoinZero ? !!v : false) continue;
    const int x = (int)(i % sz.x), y = (int)((i / sz.x) % sz.y), z = (int)(i / ((int64_t)sz.x * sz.y));
    for (int k = 0; k < nnb; ++k) {
      const int zz = z + kNb[k][0], yy = y + kNb[k][1], xx = x + kNb[k][2];
      if (zz < 0 || yy < 0 || yy >= sz.y || xx < 0 || xx >= sz.x) continue;
      const int64_t j = ((int64_t)zz * sz.y + yy) * sz.x + xx;
      if (val[j] == v) uf_unite(P, (uint32_t)i, (uint32_t)j);
    }
  }
}
