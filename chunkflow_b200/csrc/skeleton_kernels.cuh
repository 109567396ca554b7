// Device code of `skeletonize` (a TEASAR skeleton of every object of a segmentation chunk), restated in
// oracle/skeleton_oracle.py, which every kernel here follows bit for bit: float64 throughout, every multiply and add rounded on
// its own (__dmul_rn / __dadd_rn; a division or a square root is correctly rounded on its own).
// NOT a stand-alone header: skeleton.cu includes it inside the library's anonymous namespace (after `kSkThreads`);
// tests/host_emulation/skeleton_emulation.cpp compiles skeleton.cu for the host behind the one-lane CUDA shim, so every loop
// over threads or blocks is a stride loop that one lane can walk alone.
#pragma once

constexpr uint32_t kSkNone = 0xFFFFFFFFu;   // "no object" / "no index" (a chunk has fewer than 2^32 voxels)
constexpr int kSkTile = 8;                  // relaxation tiles: 8^3 voxels and a one-voxel halo
constexpr int kSkHalo = kSkTile + 2;
constexpr int kSkRows = 32;                 // x pass: rows per block, staged through shared memory 32 x positions at a time

struct SkGeom {
  int64_t Z, Y, X, n;
  double w[3];        // voxel size z, y, x
  double len[27];     // physical length of the offset (dz, dy, dx) + 1 as a base-3 number (13 distinct values)
};

struct SkParams {
  double scale, cst, pdrf_scale;
  int exponent;
};

__host__ __device__ __forceinline__ uint32_t sk_float_bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return u;
#endif
}

__host__ __device__ __forceinline__ float sk_bits_float(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  std::memcpy(&f, &u, 4);
  return f;
#endif
}

__host__ __device__ __forceinline__ unsigned long long sk_double_bits(double d) {
#ifdef __CUDA_ARCH__
  return (unsigned long long)__double_as_longlong(d);
#else
  unsigned long long u;
  std::memcpy(&u, &d, 8);
  return u;
#endif
}

__device__ __forceinline__ double sk_sq(double a) { return __dmul_rn(a, a); }

template <typename T>
__device__ __forceinline__ unsigned long long sk_id(const T* __restrict__ seg, int64_t i) { return (unsigned long long)seg[i]; }

__device__ __forceinline__ bool sk_skipped(const unsigned long long* __restrict__ skip, int64_t n, unsigned long long id) {
  int64_t lo = 0, hi = n;   // skip is sorted
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (skip[mid] < id) lo = mid + 1; else hi = mid;
  }
  return lo < n && skip[lo] == id;
}

// ---- DBF, x pass: run distance k = min(q - a + 1, b - q) of every voxel of a run [a, b) of one non-zero id (0 for id 0).
// A block stages kSkRows consecutive rows 32 x positions at a time (coalesced loads), then each row is walked by one thread:
// forward for the distance to the run's start, backward for the distance to its end.
template <typename T>
__global__ void __launch_bounds__(kSkRows) sk_edt_x_kernel(const T* __restrict__ seg, SkGeom g, uint32_t* __restrict__ kx) {
  __shared__ unsigned long long s_id[kSkRows][33], s_prev[kSkRows];
  __shared__ uint32_t s_k[kSkRows][33], s_run[kSkRows];   // s_prev, s_run: each row's last id and run length so far
  const int64_t rows = g.Z * g.Y, groups = (rows + kSkRows - 1) / kSkRows, tiles = (g.X + 31) / 32;
  for (int64_t grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    const int64_t r0 = grp * kSkRows;
    const int nr = (int)min((int64_t)kSkRows, rows - r0);
    for (int dir = 0; dir < 2; ++dir) {   // 0: left to right, 1: right to left
      for (int64_t tt = 0; tt < tiles; ++tt) {
        const int64_t x0 = (dir ? tiles - 1 - tt : tt) * 32;
        const int nx = (int)min((int64_t)32, g.X - x0);
        __syncthreads();
        for (int e = threadIdx.x; e < kSkRows * 32; e += blockDim.x) {
          const int r = e >> 5, c = e & 31;
          if (r < nr && c < nx) {
            const int64_t i = (r0 + r) * g.X + x0 + c;
            s_id[r][c] = sk_id(seg, i);
            if (dir) s_k[r][c] = kx[i];
          }
        }
        __syncthreads();
        for (int r = threadIdx.x; r < nr; r += blockDim.x) {
          uint32_t run = tt ? s_run[r] : 0u;
          unsigned long long prev = tt ? s_prev[r] : 0ULL;
          for (int cc = 0; cc < nx; ++cc) {
            const int c = dir ? nx - 1 - cc : cc;
            const unsigned long long id = s_id[r][c];
            run = (cc == 0 && tt == 0) || id != prev ? 1u : run + 1u;
            prev = id;
            s_k[r][c] = id == 0ULL ? 0u : (dir ? min(s_k[r][c], run) : run);
          }
          s_run[r] = run;
          s_prev[r] = prev;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < kSkRows * 32; e += blockDim.x) {
          const int r = e >> 5, c = e & 31;
          if (r < nr && c < nx) kx[(r0 + r) * g.X + x0 + c] = s_k[r][c];
        }
      }
    }
  }
}

// ---- DBF, y and z passes: one thread per column, a warp on 32 adjacent x.  Each run [a, b) of one non-zero id:
// Felzenszwalb-Huttenlocher's lower envelope of its own sites, then the minimum with the two outside neighbours at distance 0.
// The envelope's stack lives in global memory (`vstack`, at the run's own positions of the column) and site values are read
// again for every intersection test.  A warp's accesses are one contiguous segment only while its 32 columns step through runs
// and stack pops in lockstep (coherent objects); elsewhere the threads diverge and the accesses scatter, which is why these
// passes reach a few per cent of HBM bandwidth.  Staging the columns in shared memory is left for later.
template <bool kZ>
__device__ __forceinline__ double sk_site(const uint32_t* __restrict__ kx, const double* __restrict__ d2, const SkGeom& g, int64_t i) {
  if (kZ) return d2[i];
  return sk_sq(__dmul_rn((double)kx[i], g.w[2]));
}

template <bool kZ>
__device__ __forceinline__ double sk_meet(const uint32_t* __restrict__ kx, const double* __restrict__ d2, const SkGeom& g, int64_t base,
                                          int64_t step, int64_t p, int64_t q, double w) {
  const double qw = __dmul_rn((double)q, w), pw = __dmul_rn((double)p, w);
  const double num = __dadd_rn(__dadd_rn(sk_site<kZ>(kx, d2, g, base + q * step), sk_sq(qw)),
                               -__dadd_rn(sk_site<kZ>(kx, d2, g, base + p * step), sk_sq(pw)));
  return num / __dmul_rn(__dmul_rn(w, w), (double)(2 * (q - p)));
}

template <typename T, bool kZ>
__global__ void __launch_bounds__(kSkThreads) sk_edt_col_kernel(const T* __restrict__ seg, SkGeom g, const uint32_t* __restrict__ kx,
                                                                 double* __restrict__ d2, uint32_t* __restrict__ vstack,
                                                                 float* __restrict__ dbf) {
  const int64_t other = kZ ? g.Y : g.Z;       // columns: (z, x) for y, (y, x) for z
  const int64_t L = kZ ? g.Z : g.Y;
  const int64_t step = kZ ? g.Y * g.X : g.X;
  const double w = kZ ? g.w[0] : g.w[1];
  const int64_t cols = other * g.X, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += stride) {
    const int64_t x = c % g.X, o = c / g.X;
    const int64_t base = kZ ? o * g.X + x : o * g.Y * g.X + x;
    int64_t a = 0;
    while (a < L) {
      const unsigned long long id = sk_id(seg, base + a * step);
      int64_t b = a + 1;
      while (b < L && sk_id(seg, base + b * step) == id) ++b;
      if (id == 0ULL) {
        for (int64_t q = a; q < b; ++q) {
          if (kZ) dbf[base + q * step] = 0.f; else d2[base + q * step] = 0.0;
        }
        a = b;
        continue;
      }
      // the envelope: vstack[base + (a + k) step] = k-th site
      int64_t top = 0;
      vstack[base + a * step] = (uint32_t)a;
      for (int64_t q = a + 1; q < b; ++q) {
        while (top > 0) {
          const int64_t v1 = vstack[base + (a + top) * step], v0 = vstack[base + (a + top - 1) * step];
          if (sk_meet<kZ>(kx, d2, g, base, step, v1, q, w) <= sk_meet<kZ>(kx, d2, g, base, step, v0, v1, w)) --top;
          else break;
        }
        ++top;
        vstack[base + (a + top) * step] = (uint32_t)q;
      }
      // kZ reads d2 (the y pass) and writes dbf; the y pass reads kx and writes d2: a site's value is never overwritten early
      int64_t k = 0;
      for (int64_t q = a; q < b; ++q) {
        while (k < top && sk_meet<kZ>(kx, d2, g, base, step, vstack[base + (a + k) * step], vstack[base + (a + k + 1) * step], w) <
                              (double)q)
          ++k;
        const int64_t v = vstack[base + (a + k) * step];
        const double lo = sk_sq(__dmul_rn((double)(q - a + 1), w)), hi = sk_sq(__dmul_rn((double)(b - q), w));
        double best = lo < hi ? lo : hi;
        const double env = __dadd_rn(sk_site<kZ>(kx, d2, g, base + v * step), sk_sq(__dmul_rn((double)(q - v), w)));
        if (env < best) best = env;
        if (kZ) dbf[base + q * step] = __double2float_rn(sqrt(best));
        else d2[base + q * step] = best;
      }
      a = b;
    }
  }
}

// ---- objects: union-find roots (union_find.cuh) flattened, voxels counted per root ----
__global__ void __launch_bounds__(kSkThreads) sk_init_kernel(uint32_t* __restrict__ P, uint32_t* __restrict__ count, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    P[i] = (uint32_t)i;
    count[i] = 0u;
  }
}

template <typename T>
__global__ void __launch_bounds__(kSkThreads) sk_flatten_kernel(const T* __restrict__ seg, uint32_t* __restrict__ P, uint32_t* __restrict__ count,
                                                                int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (sk_id(seg, i) == 0ULL) continue;
    const uint32_t r = uf_find(P, (uint32_t)i);
    P[i] = r;
    atomicAdd(&count[r], 1u);
  }
}

// a root is kept when its id is not skipped and its component has at least dust_threshold voxels
template <typename T>
__device__ __forceinline__ bool sk_kept(const T* __restrict__ seg, const uint32_t* __restrict__ count, const unsigned long long* __restrict__ skip,
                                        int64_t num_skip, uint64_t dust, uint32_t r) {
  const unsigned long long id = sk_id(seg, r);
  return id != 0ULL && (uint64_t)count[r] >= dust && !(num_skip && sk_skipped(skip, num_skip, id));
}

template <typename T>
__global__ void __launch_bounds__(kSkThreads) sk_root_flags_kernel(const T* __restrict__ seg, const uint32_t* __restrict__ P,
                                                                   const uint32_t* __restrict__ count, const unsigned long long* __restrict__ skip,
                                                                   int64_t num_skip, uint64_t dust, int64_t n, uint32_t* __restrict__ flag,
                                                                   unsigned long long* __restrict__ kept_voxels) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool root = sk_id(seg, i) != 0ULL && P[i] == (uint32_t)i && sk_kept(seg, count, skip, num_skip, dust, (uint32_t)i);
    flag[i] = root ? 1u : 0u;
    if (root) atomicAdd(kept_voxels, (unsigned long long)count[i]);
  }
}

// obj[i] = the object (rank of its kept root) of every voxel, kSkNone elsewhere
template <typename T>
__global__ void __launch_bounds__(kSkThreads) sk_objects_kernel(const T* __restrict__ seg, const uint32_t* __restrict__ P,
                                                                const uint32_t* __restrict__ count, const unsigned long long* __restrict__ skip,
                                                                int64_t num_skip, uint64_t dust, const uint32_t* __restrict__ rank, int64_t n,
                                                                uint32_t* __restrict__ obj) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint32_t o = kSkNone;
    if (sk_id(seg, i) != 0ULL) {
      const uint32_t r = P[i];
      if (sk_kept(seg, count, skip, num_skip, dust, r)) o = rank[r];
    }
    obj[i] = o;
  }
}

// ---- per object: voxel count (-> starts), root key, bounding box ----
__global__ void __launch_bounds__(kSkThreads) sk_object_init_kernel(const uint32_t* __restrict__ P, const uint32_t* __restrict__ obj,
                                                                    const uint32_t* __restrict__ count, int64_t n, uint32_t* __restrict__ start,
                                                                    unsigned long long* __restrict__ key, int* __restrict__ bbox, int64_t K) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < K; o += stride) {
    key[o] = 0ULL;
    for (int k = 0; k < 3; ++k) { bbox[6 * o + k] = INT32_MAX; bbox[6 * o + 3 + k] = -1; }
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    if (obj[i] != kSkNone && P[i] == (uint32_t)i) start[obj[i]] = count[i];
}

// the root: one atomicMax per voxel on (DBF bits << 32 | ~index): the largest DBF, ties to the smallest index
__global__ void __launch_bounds__(kSkThreads) sk_roots_kernel(const uint32_t* __restrict__ obj, const float* __restrict__ dbf, SkGeom g,
                                                              unsigned long long* __restrict__ key, int* __restrict__ bbox) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += stride) {
    const uint32_t o = obj[i];
    if (o == kSkNone) continue;
    const unsigned long long k = ((unsigned long long)sk_float_bits(dbf[i]) << 32) | (unsigned long long)(~(uint32_t)i);
    if (k > key[o]) atomicMax(&key[o], k);
    const int c[3] = {(int)(i / (g.Y * g.X)), (int)((i / g.X) % g.Y), (int)(i % g.X)};
    for (int a = 0; a < 3; ++a) {
      if (c[a] < bbox[6 * o + a]) atomicMin(&bbox[6 * o + a], c[a]);
      if (c[a] > bbox[6 * o + 3 + a]) atomicMax(&bbox[6 * o + 3 + a], c[a]);
    }
  }
}

__device__ __forceinline__ uint32_t sk_root(unsigned long long key) { return ~(uint32_t)(key & 0xFFFFFFFFULL); }

__device__ __forceinline__ double sk_pdrf(float dbf_v, unsigned long long key, const SkParams& prm) {
  const double t = __dadd_rn(1.0, -((double)dbf_v / (double)sk_bits_float((uint32_t)(key >> 32))));
  double p = t;
  for (int k = 1; k < prm.exponent; ++k) p = __dmul_rn(p, t);
  return __dadd_rn(__dmul_rn(prm.pdrf_scale, p), 1.0);
}

// ---- D: infinity everywhere, 0 at the roots, whose tiles are the first to relax ----
__global__ void __launch_bounds__(kSkThreads) sk_d_init_kernel(double* __restrict__ D, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) D[i] = (double)INFINITY;
}

struct SkTiles {
  int64_t t[3];   // tiles along z, y, x
  int64_t count;
};

__global__ void __launch_bounds__(kSkThreads) sk_d_roots_kernel(const unsigned long long* __restrict__ key, int64_t K, SkGeom g, SkTiles tl,
                                                                double* __restrict__ D, uint32_t* __restrict__ dirty) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < K; o += stride) {
    const int64_t r = sk_root(key[o]);
    D[r] = 0.0;
    const int64_t z = r / (g.Y * g.X), y = (r / g.X) % g.Y, x = r % g.X;
    dirty[((z / kSkTile) * tl.t[1] + y / kSkTile) * tl.t[2] + x / kSkTile] = 1u;
  }
}

// One sweep of block-tiled relaxation: every tile next to a tile that changed in the last sweep loads itself and a one-voxel
// halo, relaxes D(v) = min(D(v), D(u) + len(u -> v) PDRF(v)) over the 26 neighbours of its own object until nothing changes
// in the tile, and writes back what changed.  Values read while other tiles write are upper bounds of the fixed point, so the
// order does not matter (DESIGN.md f10); a sweep without a change anywhere ends the relaxation.
__global__ void __launch_bounds__(kSkThreads) sk_relax_kernel(const uint32_t* __restrict__ obj, const float* __restrict__ dbf, SkGeom g,
                                                              SkParams prm, const unsigned long long* __restrict__ key, SkTiles tl,
                                                              double* __restrict__ D, const uint32_t* __restrict__ dirty,
                                                              uint32_t* __restrict__ next, uint32_t* __restrict__ changed) {
  __shared__ double s_d[kSkHalo * kSkHalo * kSkHalo];
  __shared__ uint32_t s_o[kSkHalo * kSkHalo * kSkHalo];
  __shared__ double s_p[kSkTile * kSkTile * kSkTile];
  __shared__ int s_changed, s_any;
  for (int64_t t = blockIdx.x; t < tl.count; t += gridDim.x) {
    const int64_t tz = t / (tl.t[1] * tl.t[2]), ty = (t / tl.t[2]) % tl.t[1], tx = t % tl.t[2];
    bool run = false;
    for (int64_t dz = -1; dz <= 1; ++dz)
      for (int64_t dy = -1; dy <= 1; ++dy)
        for (int64_t dx = -1; dx <= 1; ++dx) {
          const int64_t a = tz + dz, b = ty + dy, c = tx + dx;
          if (a >= 0 && b >= 0 && c >= 0 && a < tl.t[0] && b < tl.t[1] && c < tl.t[2] && dirty[(a * tl.t[1] + b) * tl.t[2] + c]) run = true;
        }
    if (!run) continue;   // the same for every thread of the block
    const int64_t z0 = tz * kSkTile - 1, y0 = ty * kSkTile - 1, x0 = tx * kSkTile - 1;
    __syncthreads();
    for (int e = threadIdx.x; e < kSkHalo * kSkHalo * kSkHalo; e += blockDim.x) {
      const int64_t z = z0 + e / (kSkHalo * kSkHalo), y = y0 + (e / kSkHalo) % kSkHalo, x = x0 + e % kSkHalo;
      uint32_t o = kSkNone;
      double d = (double)INFINITY;
      if (z >= 0 && y >= 0 && x >= 0 && z < g.Z && y < g.Y && x < g.X) {
        const int64_t i = (z * g.Y + y) * g.X + x;
        o = obj[i];
        if (o != kSkNone) d = D[i];
      }
      s_o[e] = o;
      s_d[e] = d;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kSkTile * kSkTile * kSkTile; e += blockDim.x) {
      const int h = ((e / 64 + 1) * kSkHalo + (e / 8) % 8 + 1) * kSkHalo + e % 8 + 1;
      const int64_t z = z0 + 1 + e / 64, y = y0 + 1 + (e / 8) % 8, x = x0 + 1 + e % 8;
      s_p[e] = s_o[h] == kSkNone ? 0.0 : sk_pdrf(dbf[(z * g.Y + y) * g.X + x], key[s_o[h]], prm);
    }
    if (threadIdx.x == 0) s_any = 0;
    for (;;) {
      __syncthreads();
      if (threadIdx.x == 0) s_changed = 0;
      __syncthreads();
      for (int e = threadIdx.x; e < kSkTile * kSkTile * kSkTile; e += blockDim.x) {
        const int h = ((e / 64 + 1) * kSkHalo + (e / 8) % 8 + 1) * kSkHalo + e % 8 + 1;
        const uint32_t o = s_o[h];
        if (o == kSkNone) continue;
        double best = s_d[h];
        for (int k = 0; k < 27; ++k) {
          if (k == 13) continue;
          const int u = h + ((k / 9) - 1) * kSkHalo * kSkHalo + ((k / 3) % 3 - 1) * kSkHalo + (k % 3 - 1);
          if (s_o[u] != o) continue;
          const double c = __dadd_rn(s_d[u], __dmul_rn(g.len[k], s_p[e]));
          if (c < best) best = c;
        }
        if (best < s_d[h]) {
          s_d[h] = best;
          s_changed = 1;
        }
      }
      __syncthreads();
      if (!s_changed) break;
      if (threadIdx.x == 0) s_any = 1;
    }
    if (s_any) {
      for (int e = threadIdx.x; e < kSkTile * kSkTile * kSkTile; e += blockDim.x) {
        const int h = ((e / 64 + 1) * kSkHalo + (e / 8) % 8 + 1) * kSkHalo + e % 8 + 1;
        const int64_t z = z0 + 1 + e / 64, y = y0 + 1 + (e / 8) % 8, x = x0 + 1 + e % 8;
        if (s_o[h] == kSkNone || z >= g.Z || y >= g.Y || x >= g.X) continue;
        const int64_t i = (z * g.Y + y) * g.X + x;
        if (s_d[h] < D[i]) D[i] = s_d[h];
      }
      if (threadIdx.x == 0) {
        next[t] = 1u;
        *changed = 1u;
      }
    }
  }
}

// ---- Parent(v): the neighbour of the same object attaining D(v), ties to the smallest index; the roots point at themselves ----
__global__ void __launch_bounds__(kSkThreads) sk_parent_kernel(const uint32_t* __restrict__ obj, const float* __restrict__ dbf, SkGeom g,
                                                               SkParams prm, const unsigned long long* __restrict__ key,
                                                               const double* __restrict__ D, uint32_t* __restrict__ parent) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += stride) {
    const uint32_t o = obj[i];
    if (o == kSkNone) continue;
    if (sk_root(key[o]) == (uint32_t)i) { parent[i] = (uint32_t)i; continue; }
    const double p = sk_pdrf(dbf[i], key[o], prm);
    const int64_t z = i / (g.Y * g.X), y = (i / g.X) % g.Y, x = i % g.X;
    double best = (double)INFINITY;
    uint32_t bu = kSkNone;
#pragma unroll 1
    for (int k = 0; k < 27; ++k) {   // ascending offset = ascending index
      if (k == 13) continue;
      const int64_t zz = z + k / 9 - 1, yy = y + (k / 3) % 3 - 1, xx = x + k % 3 - 1;
      if (zz < 0 || yy < 0 || xx < 0 || zz >= g.Z || yy >= g.Y || xx >= g.X) continue;
      const int64_t u = (zz * g.Y + yy) * g.X + xx;
      if (obj[u] != o) continue;
      const double c = __dadd_rn(D[u], __dmul_rn(g.len[k], p));
      if (c < best) { best = c; bu = (uint32_t)u; }
    }
    parent[i] = bu;
  }
}

// ---- the sort: (~D bits, index) of every voxel of an object, compacted in index order; then the object replaces the key ----
__global__ void __launch_bounds__(kSkThreads) sk_flag_kernel(const uint32_t* __restrict__ obj, int64_t n, uint32_t* __restrict__ flag) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) flag[i] = obj[i] != kSkNone ? 1u : 0u;
}

__global__ void __launch_bounds__(kSkThreads) sk_emit_kernel(const uint32_t* __restrict__ obj, const double* __restrict__ D,
                                                             const uint32_t* __restrict__ pos, int64_t n, unsigned long long* __restrict__ ids,
                                                             unsigned long long* __restrict__ vals) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (obj[i] == kSkNone) continue;
    ids[pos[i]] = ~sk_double_bits(D[i]);   // D >= 0: descending D is ascending ~bits
    vals[pos[i]] = (unsigned long long)i;
  }
}

__global__ void __launch_bounds__(kSkThreads) sk_object_keys_kernel(const uint32_t* __restrict__ obj, const unsigned long long* __restrict__ vals,
                                                                    int64_t m, unsigned long long* __restrict__ ids) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) ids[j] = obj[vals[j]];
}

// ---- rounds ----
// counters: 0 path voxels so far, 1 first path voxel of this round, 2 "a target was found", 3 paths so far, 4 a broken Parent chain
constexpr int kSkCounters = 8;

__global__ void sk_round_begin_kernel(unsigned long long* __restrict__ counters) {
  counters[1] = counters[0];
  counters[2] = 0ULL;
}

// one thread per object: move the cursor past invalidated voxels; the first valid one is the target; trace it along Parent to
// the root or to the skeleton, appending the new voxels to the path list.  The parameter rules keep D finite and strictly
// increasing, so every chain ends at the root within the object's size; a chain that does not (no Parent, or longer than the
// object) is not followed: counters[4] is set and the host stops with an error.
__global__ void __launch_bounds__(kSkThreads) sk_trace_kernel(const unsigned long long* __restrict__ vals, const uint32_t* __restrict__ start,
                                                              uint32_t* __restrict__ cursor, int64_t K, const uint8_t* __restrict__ valid,
                                                              const uint32_t* __restrict__ parent, uint8_t* __restrict__ on,
                                                              uint32_t* __restrict__ path, unsigned long long* __restrict__ counters) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < K; o += stride) {
    uint32_t c = cursor[o];
    const uint32_t e = start[o + 1];
    while (c < e && !valid[vals[c]]) ++c;
    cursor[o] = c;
    if (c == e) continue;
    const uint32_t t = (uint32_t)vals[c], size = e - start[o];
    uint32_t len = 0;
    bool broken = false;
    for (uint32_t v = t; !on[v]; v = parent[v]) {
      if (parent[v] == kSkNone || ++len > size) {
        broken = true;
        break;
      }
      if (parent[v] == v) break;
    }
    if (broken) {
      counters[4] = 1ULL;
      continue;
    }
    unsigned long long j = atomicAdd(&counters[0], (unsigned long long)len);
    for (uint32_t v = t; !on[v]; v = parent[v]) {
      path[j++] = v;
      on[v] = 1;
      if (parent[v] == v) break;
    }
    counters[2] = 1ULL;
    atomicAdd(&counters[3], 1ULL);
  }
}

// CTAs over (path voxel of this round, z slab of its ball's bounding box clamped to the object's): every voxel of the object
// within r = scale DBF(p) + const of path voxel p is no longer a target
__global__ void __launch_bounds__(kSkThreads) sk_invalidate_kernel(const uint32_t* __restrict__ path, const unsigned long long* __restrict__ counters,
                                                                   const uint32_t* __restrict__ obj, const float* __restrict__ dbf, SkGeom g,
                                                                   SkParams prm, const int* __restrict__ bbox, uint8_t* __restrict__ valid) {
  const unsigned long long begin = counters[1], end = counters[0];
  for (unsigned long long j = begin + blockIdx.x; j < end; j += gridDim.x) {
    const int64_t p = path[j];
    const uint32_t o = obj[p];
    const int64_t pc[3] = {p / (g.Y * g.X), (p / g.X) % g.Y, p % g.X};
    const double r = __dadd_rn(__dmul_rn(prm.scale, (double)dbf[p]), prm.cst), r2 = sk_sq(r);
    int64_t lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
      const double q = r / g.w[a];   // the exact test below decides; a chunk axis is shorter than 2^31
      const int64_t ext = q < 4.0e9 ? (int64_t)floor(q) + 1 : (int64_t)4000000000LL;
      lo[a] = max(pc[a] - ext, (int64_t)bbox[6 * o + a]);
      hi[a] = min(pc[a] + ext, (int64_t)bbox[6 * o + 3 + a]);
    }
    const int64_t ny = hi[1] - lo[1] + 1, nx = hi[2] - lo[2] + 1;
    for (int64_t z = lo[0] + blockIdx.y; z <= hi[0]; z += gridDim.y) {
      const double dz = sk_sq(__dmul_rn((double)(z - pc[0]), g.w[0]));
      for (int64_t e = threadIdx.x; e < ny * nx; e += blockDim.x) {
        const int64_t y = lo[1] + e / nx, x = lo[2] + e % nx;
        const int64_t i = (z * g.Y + y) * g.X + x;
        if (obj[i] != o || !valid[i]) continue;
        const double d2 = __dadd_rn(__dadd_rn(dz, sk_sq(__dmul_rn((double)(y - pc[1]), g.w[1]))), sk_sq(__dmul_rn((double)(x - pc[2]), g.w[2])));
        if (d2 <= r2) valid[i] = 0;
      }
    }
  }
}

// ---- the skeleton voxels for the host: (id, DBF bits << 32 | Parent) of every path voxel ----
template <typename T>
__global__ void __launch_bounds__(kSkThreads) sk_gather_kernel(const T* __restrict__ seg, const uint32_t* __restrict__ path, int64_t S,
                                                               const float* __restrict__ dbf, const uint32_t* __restrict__ parent,
                                                               unsigned long long* __restrict__ ids, unsigned long long* __restrict__ vals) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < S; j += stride) {
    const uint32_t p = path[j];
    ids[j] = sk_id(seg, p);
    vals[j] = ((unsigned long long)sk_float_bits(dbf[p]) << 32) | parent[p];
  }
}
