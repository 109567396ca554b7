// wgmma / TMA implicit-GEMM 3x3x3 convolution for sm_90a.  See kernels_conv.cuh for the activation
// layout.  One CTA owns a (batch, y-tile, x-tile) column of the patch and marches along z with a ring
// of three z-planes in shared memory:
//
//   warp 0       : A producer  -- one TMA box per z-plane (halo rows/cols, zero fill outside the patch)
//   warp 1       : B producer  -- the packed weights of one tap per stage via cp.async.bulk
//   warpgroups 1, 2: consumers -- per z-plane job: 27 taps x K steps x MT tiles of wgmma.mma_async
//                                 (M = 64 positions, N = Cout or 2 * Cout, fp32 accumulators in registers),
//                                 then the epilogue: bias, ReLU, number format, 16-byte stores
//
// A tile is a dense run of 64 positions of the (TY + 2) x pitch halo plane; a tap (dy, dx) is a plain
// +16 B x (dy * pitch + dx) on the descriptor start address.  Positions in the two halo columns of a row
// compute junk that the epilogue drops.
//
// Number formats (act_format.cuh), all accumulating in fp32:
//   f16   : acc = A * W                                  (one fp16 product)
//   f16x2 : acc = A_hi * [W_hi | W_lo] + A_lo * W_hi     (N = 2 Cout for the first product; the halves are added)
//   f16f8 : acc = H * WH + [A8 | L8] * [WL8 ; W8]        (fp16 K = 16 plus e4m3 K = 32 into a second accumulator half),
//           scaled by 1 / (alpha beta)
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "act_format.cuh"
#include "chunkflow_b200.h"
#include "kernels_conv.cuh"
#include "wgmma_ops.cuh"

namespace cfb {

namespace {

// ------------------------------------------------------------------------------------------
// PTX helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a launch failure (trap) instead of a hung GPU.  The bound (~1 min at 2 GHz) is far
// beyond any legitimate wait, including time-slicing with other contexts on a shared GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 120000000000ll) {
      printf("chunkflow_b200: mbarrier timeout (block %d thread %d bar 0x%x parity %u)\n", (int)blockIdx.x,
             (int)threadIdx.x, bar, parity);
      __trap();
    }
  }
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across an asynchronous wgmma
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void named_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// K-major, no-swizzle shared memory matrix descriptor (sm_90 wgmma), 64 bits:
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4 (between the two core matrices along K)
//   [32,46) stride byte offset >> 4 (between 8-row groups)   [62,64) swizzle = 0.
// Core matrix = 8 rows x 16 bytes; SBO is always 128 B here (8 consecutive voxel records / weight rows).
__device__ __forceinline__ uint64_t gdesc(uint32_t addr, uint32_t lbo) {
  return (uint64_t)((addr >> 4) & 0x3fffu) | ((uint64_t)((lbo >> 4) & 0x3fffu) << 16) | ((uint64_t)8u << 32);
}

// ReLU that lets NaN through like torch.relu (fmaxf(NaN, 0) would return 0 and hide a broken weight from the range check)
__device__ __forceinline__ float relu_nan(float v) { return v < 0.f ? 0.f : v; }

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Fused network tail for the last 3x3x3 layer (Cout = 16): 1x1x1 head + sigmoid + crop + bump mask +
// red.global.add into the output chunk, straight from the fp32 accumulator values.
struct FusedTail {
  const float* head_w;   // (channels, 16) first rows of the head weight
  const float* head_b;   // (channels)
  const PatchPos* patches;
  const float* mask;     // (op.z, op.y, op.x)
  float* out;            // (channels, os.z, os.y, os.x)
  int channels;
  Int3 op, crop, os;
  float scale;
};

template <int COUT, bool SPLIT>
__device__ __forceinline__ void store_cp8_16(const float (&v)[16], int cb, int b, size_t vox, size_t plane_vox,
                                             uint4* __restrict__ out16) {
  constexpr int P = SPLIT ? 2 : 1;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int chunk = cb * 2 + h;
    float hi[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) hi[i] = __half2float(__float2half_rn(v[h * 8 + i]));
    const size_t plane = ((size_t)b * (COUT / 8) + chunk) * P;
    out16[plane * plane_vox + vox] = make_uint4(pack_half2(hi[0], hi[1]), pack_half2(hi[2], hi[3]),
                                                pack_half2(hi[4], hi[5]), pack_half2(hi[6], hi[7]));
    if (SPLIT) {
      float lo[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) lo[i] = v[h * 8 + i] - hi[i];
      out16[(plane + 1) * plane_vox + vox] = make_uint4(pack_half2(lo[0], lo[1]), pack_half2(lo[2], lo[3]),
                                                        pack_half2(lo[4], lo[5]), pack_half2(lo[6], lo[7]));
    }
  }
}

// f16f8 format: 16 channels (one K step) of a voxel -> H 0..7, H 8..15, A8 0..15, L8 0..15 records
template <int COUT>
__device__ __forceinline__ void store_cp8_16_f8(const float (&v)[16], int cb, int b, size_t vox, size_t plane_vox,
                                                uint4* __restrict__ out16) {
  uint4 h0, h1, a8, l8;
  af_encode16(v, h0, h1, a8, l8);
  const size_t plane = ((size_t)b * (COUT / 8) + cb * 2) * 2;  // (chunk 2cb, part 0)
  out16[plane * plane_vox + vox] = h0;
  out16[(plane + 1) * plane_vox + vox] = a8;
  out16[(plane + 2) * plane_vox + vox] = h1;
  out16[(plane + 3) * plane_vox + vox] = l8;
}

__device__ __forceinline__ void head_blend_16(const float (&v)[16], const FusedTail& t, const float* __restrict__ s_head,
                                              const PatchPos& pp, int z, int y, int x) {
  const int oz = z - t.crop.z, oy = y - t.crop.y, ox = x - t.crop.x;  // coordinates in the cropped output patch
  if (oz < 0 || oz >= t.op.z || oy < 0 || oy >= t.op.y || ox < 0 || ox >= t.op.x) return;
  int sy = oy, sx = ox;
  if (pp.flags) tta_map(pp.flags, t.op.y, t.op.x, oy, ox, sy, sx);  // augmented variant: write back un-transformed
  const int gz = pp.oz + oz, gy = pp.oy + sy, gx = pp.ox + sx;
  if (gz < 0 || gz >= t.os.z || gy < 0 || gy >= t.os.y || gx < 0 || gx >= t.os.x) return;  // clipped by the chunk
  const float m = __ldg(t.mask + ((size_t)oz * t.op.y + oy) * t.op.x + ox) * t.scale;
  float* dst = t.out + ((size_t)gz * t.os.y + gy) * t.os.x + gx;
  const size_t out_vol = (size_t)t.os.z * t.os.y * t.os.x;
  if (t.channels == 3) {
    // the affinity head: three independent FMA chains; sigmoid with ex2.approx / rcp.approx (~1e-7 of the exact value,
    // the tolerance of this path is 1e-3)
    float a0 = s_head[48], a1 = s_head[49], a2 = s_head[50];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      a0 = fmaf(v[k], s_head[k], a0);
      a1 = fmaf(v[k], s_head[16 + k], a1);
      a2 = fmaf(v[k], s_head[32 + k], a2);
    }
    float s0 = __fdividef(m, 1.0f + __expf(-a0)), s1 = __fdividef(m, 1.0f + __expf(-a1)), s2 = __fdividef(m, 1.0f + __expf(-a2));
    if (pp.flags & kTtaChannelSym) {  // reference-literal --augment: the variant plus its channel-reversed copy
      const float e = s0 + s2;
      s0 = e; s2 = e; s1 += s1;
    }
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst), "f"(s0) : "memory");
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst + out_vol), "f"(s1) : "memory");
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst + 2 * out_vol), "f"(s2) : "memory");
    return;
  }
  float sig[8];
#pragma unroll
  for (int co = 0; co < 8; ++co) {
    if (co < t.channels) {
      float acc = s_head[t.channels * 16 + co];
#pragma unroll
      for (int k = 0; k < 16; ++k) acc = fmaf(v[k], s_head[co * 16 + k], acc);
      sig[co] = __fdiv_rn(1.0f, 1.0f + expf(-acc));
    }
  }
#pragma unroll
  for (int co = 0; co < 8; ++co) {
    if (co < t.channels) {
      float o = sig[co];
      if (pp.flags & kTtaChannelSym) {
#pragma unroll
        for (int c2 = 0; c2 < 8; ++c2) if (c2 == t.channels - 1 - co) o += sig[c2];
      }
      asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst + (size_t)co * out_vol), "f"(o * m) : "memory");
    }
  }
}

struct WgConvParams {
  int Z, Y, X;
  int XT, TY, pitch, G;    // G: M tiles of 64 positions that cover the TY x pitch output positions
  int tiles_x, tiles_y;
  int planes_a, planes_b;  // 8-channel chunks of source A / source B
  uint32_t plane_stride;   // bytes of one (TY+2) x pitch x 16 B plane in smem
  uint32_t slot_stride;    // bytes of one z-plane slot (all chunk/part planes)
  const uint8_t* wpacked;  // (tap, K step) weight blocks, see pack_conv3_weights
  const float* bias;
  __half* out;
  int relu;
  float acc_scale;  // f16f8 mode: 1 / (alpha * beta), the scale the operands carry (act_format.cuh); 1 otherwise
  int bstages;      // tap stages of weights in shared memory
  int bresident;    // 1: all 27 taps stay resident (loaded once per CTA), 0: streamed through a ring
  int zblk, zblocks; // output planes per CTA and blocks per column (a CTA walks z in [zblk * block, + zblk))
  __half* out_pool; // kConvPool: (1,2,2) max-pooled copy of the output (CP8 of Z x Y/2 x X/2)
  FusedTail tail;   // used by the TAIL = true instantiations only
};

// What a kernel instantiation computes: a 3x3x3 convolution, the same with the (1,2,2) max pool of its output fused into
// the epilogue, or a transposed convolution with kernel = stride = (1,2,2) (four 1-tap GEMMs on the centre of each staged
// plane, one per output parity (y & 1, x & 1), scattered to the doubled grid).
enum ConvMode : int { kConv = 0, kConvPool = 1, kConvT = 2 };

constexpr int kRing = 3;            // z-plane ring slots
constexpr int kMaxBStages = 27;     // weight stages: one tap each
constexpr int kThreads = 384;       // producer warpgroup + two consumer warpgroups
constexpr int kConsumers = 2;
constexpr int kTailPad = 6144;      // dense M tiles read up to 63 + 2 * pitch + 2 voxel records past the last plane
constexpr int kBarBytes = (2 * kRing + 2 * kMaxBStages) * 8 + 640;  // mbarriers + head weights (fused tail)
constexpr int kMaxSmem = 232448;    // 227 KB

template <int CIN, int COUT, int FMT>
struct ConvCfg {
  static constexpr int P = FMT == kFmtF16 ? 1 : 2;
  static constexpr int NPL = P * CIN / 8;                 // planes per slot
  static constexpr int KS = CIN / 16;                     // K = 16 steps per tap
  // accumulator columns: f16x2 main product N = 2 Cout; f16f8 two Cout halves -- the e4m3 product keeps its own half because an
  // fp8 wgmma adds into its accumulator with reduced precision (the halves are summed in fp32 by the epilogue)
  static constexpr int NA = FMT == kFmtF16 ? COUT : 2 * COUT;
  static constexpr int BLK = P * 32 * COUT;               // bytes of one (tap, K step) weight block
  static constexpr int TAP = KS * BLK;                    // bytes of one weight stage
  static constexpr int MT = NA >= 128 ? 1 : (NA == 64 ? 2 : 4);  // M tiles per consumer warpgroup (<= 64 accumulator registers)
  static constexpr int SP = COUT + 4;                     // floats per row of the epilogue staging tile
};
// epilogue staging bytes: one 64-row tile per warpgroup, or (fused pooling: 2 x 2 neighbours in one place) every M tile of the CTA
template <int CIN, int COUT, int FMT, int MODE>
__host__ __device__ constexpr int stage_bytes() {
  using Cfg = ConvCfg<CIN, COUT, FMT>;
  return (MODE == kConvPool ? kConsumers * Cfg::MT : kConsumers) * 64 * Cfg::SP * 4;
}

template <int CIN, int COUT, int FMT, bool TAIL, int MODE>
__global__ void __launch_bounds__(kThreads, 1)
conv3_wgmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                   const WgConvParams p) {
  using Cfg = ConvCfg<CIN, COUT, FMT>;
  constexpr int P = Cfg::P, MT = Cfg::MT, NA = Cfg::NA;
  constexpr int NT = MODE == kConvT ? 4 : 27;  // weight taps
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);

  const int warp = threadIdx.x >> 5;
  const int zbi = blockIdx.x % p.zblocks, col = blockIdx.x / p.zblocks;
  const int tx = col % p.tiles_x;
  const int ty = (col / p.tiles_x) % p.tiles_y;
  const int b = col / (p.tiles_x * p.tiles_y);
  const int z0 = zbi * p.zblk, Z = min(p.Z - z0, p.zblk);  // this CTA's output planes: z0 .. z0 + Z - 1
  const int x0 = tx * p.XT, y0 = ty * p.TY;

  uint8_t* sA = smem;
  uint8_t* sB = smem + kRing * p.slot_stride + kTailPad;
  float* s_stage = reinterpret_cast<float*>(sB + (size_t)p.bstages * Cfg::TAP);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_stage) + stage_bytes<CIN, COUT, FMT, MODE>());
  // barrier map: [0..2] a_full, [3..5] a_empty, [6, 6+27) b_full, [33, 33+27) b_empty
  const uint32_t bar0 = smem_u32(bars);
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  constexpr int kAF = 0, kAE = kRing, kBF = 2 * kRing, kBE = 2 * kRing + kMaxBStages;
  float* s_head = reinterpret_cast<float*>(bars + kBE + kMaxBStages);
  PatchPos pp{};
  if constexpr (TAIL) {
    for (int i = threadIdx.x; i < p.tail.channels * 16; i += kThreads) s_head[i] = p.tail.head_w[i];
    for (int i = threadIdx.x; i < p.tail.channels; i += kThreads) s_head[p.tail.channels * 16 + i] = p.tail.head_b[i];
    pp = p.tail.patches[b];
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < kRing; ++i) { mbar_init(BAR(kAF + i), 1); mbar_init(BAR(kAE + i), kConsumers); }
    for (int i = 0; i < p.bstages; ++i) { mbar_init(BAR(kBF + i), 1); mbar_init(BAR(kBE + i), kConsumers); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == 0) {
    // ---------------- A producer: z-planes z0 - 1 .. z0 + Z into the ring ----------------
    if (elect_one()) {
      const uint32_t tx_bytes = (uint32_t)Cfg::NPL * p.plane_stride;
      const int plane_a0 = b * p.planes_a * P, plane_b0 = b * p.planes_b * P;
      int slot = 0;
      uint32_t use_parity = 1;  // parity of the PREVIOUS use of the slot (no wait during the first round)
      for (int q = 0; q < Z + 2; ++q, ++slot) {
        if (slot == kRing) { slot = 0; use_parity ^= 1; }
        if (q >= kRing) mbar_wait(BAR(kAE + slot), use_parity);
        mbar_expect_tx(BAR(kAF + slot), tx_bytes);
        const uint32_t dst = smem_u32(sA + (size_t)slot * p.slot_stride);
        const uint32_t dst_b = dst + (uint32_t)(p.planes_a * P) * p.plane_stride;
        // 4-D map over 8-byte elements: a record is two elements (see make_map)
        tma_load_4d(dst, &mapA, BAR(kAF + slot), 2 * (x0 - 1), y0 - 1, z0 + q - 1, plane_a0);
        if (p.planes_b > 0) tma_load_4d(dst_b, &mapB, BAR(kAF + slot), 2 * (x0 - 1), y0 - 1, z0 + q - 1, plane_b0);
      }
    }
    return;
  }
  if (warp == 1) {
    // ---------------- B producer: one tap of weights per stage, NT per z-plane job ----------------
    if (elect_one()) {
      const uint32_t nbs = (uint32_t)p.bstages;
      const uint32_t total = p.bresident ? (uint32_t)NT : (uint32_t)Z * NT;
      uint32_t st = 0, tap = 0, prev_parity = 1;
      for (uint32_t i = 0; i < total; ++i) {
        if (i >= nbs) mbar_wait(BAR(kBE + st), prev_parity);
        mbar_expect_tx(BAR(kBF + st), Cfg::TAP);
        bulk_load(smem_u32(sB + st * Cfg::TAP), p.wpacked + (size_t)tap * Cfg::TAP, Cfg::TAP, BAR(kBF + st));
        if (++st == nbs) { st = 0; prev_parity ^= 1; }
        if (++tap == (uint32_t)NT) tap = 0;
      }
    }
    return;
  }
  if (warp < 4) return;

  // ---------------- consumers ----------------
  const int cw = (warp >> 2) - 1;           // consumer warpgroup 0 / 1
  const int wtid = threadIdx.x & 127;       // thread in the warpgroup
  const bool leader = wtid == 0;
  const int g0 = cw * MT;                   // first M tile of this warpgroup
  const int ntiles = max(0, min(MT, p.G - g0));
  const uint32_t sA0 = smem_u32(sA), sB0 = smem_u32(sB);
  const uint32_t pitch = (uint32_t)p.pitch;
  const uint32_t a_lbo = (uint32_t)P * p.plane_stride;  // chunk 2k -> chunk 2k + 1 of a K step
  const bool resident = p.bresident != 0;
  const uint32_t nbs = (uint32_t)p.bstages;
  float* stage = s_stage + (MODE == kConvPool ? 0 : (size_t)cw * 64 * Cfg::SP);
  const int ty_valid = min(p.TY, p.Y - y0), xt_valid = min(p.XT, p.X - x0);
  const size_t plane_vox = (size_t)p.Z * p.Y * p.X;
  uint4* out16 = reinterpret_cast<uint4*>(p.out);

  float acc[MT][NA / 2];
  uint32_t ring_st = 0, ring_parity = 0;
  for (int zz = 0; zz < Z; ++zz) {
    const int z = z0 + zz;
#pragma unroll
    for (int g = 0; g < MT; ++g)
#pragma unroll
      for (int i = 0; i < NA / 2; ++i) acc[g][i] = 0.f;
    int prev_st = -1;
    // ---------------- epilogue: registers -> staging tile -> bias/ReLU -> number format -> HBM ----------------
    // accumulator fragment of m64nN: thread (warp w, lane l) holds rows 16 w + l / 4 (+ 8), columns 8 j + 2 (l % 4) (+ 1)
    auto epilogue = [&](int par) {
      wg_wait<0>();
#pragma unroll
      for (int g = 0; g < MT; ++g) acc_fence(acc[g]);
      if (leader && prev_st >= 0) mbar_arrive(BAR(kBE + prev_st));  // the job's last weight stage
      prev_st = -1;
      if (MODE != kConvT && leader) mbar_arrive(BAR(kAE + (zz % kRing)));  // plane z-1 is dead: the producer may refill its slot
      const int wr = (wtid >> 5) * 16 + ((wtid & 31) >> 2), wc = 2 * (wtid & 3);
      // one voxel's 16 channels from the staging rows: accumulator scale, bias, ReLU
      auto load16 = [&](int row, int cb, float (&v)[16]) {
        const float4* src = reinterpret_cast<const float4*>(stage + row * Cfg::SP + cb * 16);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 f = src[i];
          v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w;
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          v[i] = fmaf(v[i], p.acc_scale, __ldg(p.bias + cb * 16 + i));
          if (p.relu) v[i] = relu_nan(v[i]);
        }
      };
      auto store16 = [&](const float (&v)[16], int cb, size_t vox, size_t pvol, uint4* dst) {
        if constexpr (FMT == kFmtF16F8) store_cp8_16_f8<COUT>(v, cb, b, vox, pvol, dst);
        else store_cp8_16<COUT, FMT == kFmtF16x2>(v, cb, b, vox, pvol, dst);
      };
      // kConvPool stages every tile of the CTA (rows = CTA positions) before anyone reads; otherwise one tile at a time
      constexpr int NPASS = MODE == kConvPool ? 1 : MT;
      for (int pass = 0; pass < NPASS; ++pass) {
        if (MODE != kConvPool && pass >= ntiles) break;
#pragma unroll
        for (int g = 0; g < MT; ++g) {
          if (MODE == kConvPool ? g >= ntiles : g != pass) continue;
          const int row0 = MODE == kConvPool ? (g0 + g) * 64 : 0;
#pragma unroll
          for (int j = 0; j < COUT / 8; ++j) {
            float v0 = acc[g][4 * j], v1 = acc[g][4 * j + 1], v2 = acc[g][4 * j + 2], v3 = acc[g][4 * j + 3];
            if constexpr (FMT != kFmtF16) {  // + the second half (f16x2: w_lo columns of the first product; f16f8: e4m3 product)
              v0 += acc[g][COUT / 2 + 4 * j]; v1 += acc[g][COUT / 2 + 4 * j + 1];
              v2 += acc[g][COUT / 2 + 4 * j + 2]; v3 += acc[g][COUT / 2 + 4 * j + 3];
            }
            *reinterpret_cast<float2*>(stage + (row0 + wr) * Cfg::SP + 8 * j + wc) = make_float2(v0, v1);
            *reinterpret_cast<float2*>(stage + (row0 + wr + 8) * Cfg::SP + 8 * j + wc) = make_float2(v2, v3);
          }
        }
        if (MODE == kConvPool) named_sync(3, 256); else named_sync(1 + cw, 128);
        // rows handled by this pass and the threads sharing them
        const int nrows = MODE == kConvPool ? p.G * 64 : 64, tid = MODE == kConvPool ? (int)threadIdx.x - 128 : wtid;
        const int nthr = MODE == kConvPool ? 256 : 128, rowq0 = MODE == kConvPool ? 0 : (g0 + pass) * 64;
        for (int item = tid; item < nrows * (COUT / 16); item += nthr) {
          const int row = item % nrows, cb = item / nrows;
          const int qpos = rowq0 + row;
          const int r = qpos / p.pitch, col = qpos - r * p.pitch;
          if (r >= ty_valid || col >= xt_valid) continue;
          float v[16];
          load16(row, cb, v);
          if constexpr (MODE == kConvT) {  // output parity par = (oy & 1) * 2 + (ox & 1) on the doubled grid
            const int oy = 2 * (y0 + r) + (par >> 1), ox = 2 * (x0 + col) + (par & 1);
            store16(v, cb, ((size_t)z * 2 * p.Y + oy) * 2 * p.X + ox, plane_vox * 4, out16);
          } else if constexpr (TAIL) {
            head_blend_16(v, p.tail, s_head, pp, z, y0 + r, x0 + col);
          } else {
            store16(v, cb, ((size_t)z * p.Y + (y0 + r)) * p.X + (x0 + col), plane_vox, out16);
          }
        }
        if constexpr (MODE == kConvPool) {  // (1,2,2) max pool of the same values (y0, x0, TY, XT and the extents are even)
          const int PX = p.XT / 2, npool = (p.TY / 2) * PX;
          for (int item = tid; item < npool * (COUT / 16); item += nthr) {
            const int pi = item % npool, cb = item / npool;
            const int pr = pi / PX, pc = pi - pr * PX;
            if (2 * pr >= ty_valid || 2 * pc >= xt_valid) continue;
            float m[16], v[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) m[i] = -INFINITY;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              load16((2 * pr + (k >> 1)) * p.pitch + 2 * pc + (k & 1), cb, v);
#pragma unroll
              for (int i = 0; i < 16; ++i) m[i] = fmaxf(m[i], v[i]);
            }
            const size_t pvox = ((size_t)z * (p.Y / 2) + (y0 / 2 + pr)) * (p.X / 2) + (x0 / 2 + pc);
            store16(m, cb, pvox, plane_vox / 4, reinterpret_cast<uint4*>(p.out_pool));
          }
        }
        if (MODE == kConvPool) named_sync(3, 256); else named_sync(1 + cw, 128);
      }
    };
    if (MODE == kConvT && zz == 0) mbar_wait(BAR(kAF + 0), 0);  // plane z0 - 1 (unused) must have landed before its slot is freed
    // conv: 27 taps accumulate into one job; convT: the 4 output parities are 4 jobs on the centre tap of plane z
    for (int t = 0; t < NT; ++t) {
      const int dz = MODE == kConvT ? 1 : t / 9, dy = MODE == kConvT ? 1 : (t / 3) % 3, dx = MODE == kConvT ? 1 : t % 3;
      const int q = zz + dz, slot = q % kRing;
      if (MODE == kConvT ? t == 0 : (dy == 0 && dx == 0)) mbar_wait(BAR(kAF + slot), (uint32_t)(q / kRing) & 1u);
      const uint32_t a_slot = sA0 + (uint32_t)slot * p.slot_stride;
      if (MODE == kConvT && t > 0) {
#pragma unroll
        for (int g = 0; g < MT; ++g)
#pragma unroll
          for (int i = 0; i < NA / 2; ++i) acc[g][i] = 0.f;
      }
      {
        {
          const int tap = t;
          uint32_t st;
          if (resident) {
            st = (uint32_t)tap;
            if (zz == 0) mbar_wait(BAR(kBF + st), 0);  // taps arrive once
          } else {
            st = ring_st;
            mbar_wait(BAR(kBF + st), ring_parity);
            if (++ring_st == nbs) { ring_st = 0; ring_parity ^= 1; }
          }
          const uint32_t b_tap = sB0 + st * Cfg::TAP;
          const uint32_t a_tap = a_slot + (uint32_t)(dy * pitch + dx) * 16u;
#pragma unroll
          for (int g = 0; g < MT; ++g) acc_fence(acc[g]);
          wg_fence();
          // main products; accumulator accesses are ordered only between wgmma of the same shape, so the f16x2 second
          // products (same registers, different shape) wait for the first group; the f16f8 e4m3 products use their own half
#pragma unroll
          for (int ks = 0; ks < Cfg::KS; ++ks) {
            const uint32_t b_blk = b_tap + (uint32_t)ks * Cfg::BLK;
            const uint32_t a_ks = a_tap + (uint32_t)(2 * ks * P) * p.plane_stride;
#pragma unroll
            for (int g = 0; g < MT; ++g) {
              if (g < ntiles) {
                const uint32_t a = a_ks + (uint32_t)((g0 + g) * 64) * 16u;
                if constexpr (FMT == kFmtF16x2) wgmma_f16<2 * COUT>(acc[g], gdesc(a, a_lbo), gdesc(b_blk, 2 * COUT * 16), 1);
                else wgmma_f16<COUT>(reinterpret_cast<float(&)[COUT / 2]>(acc[g]), gdesc(a, a_lbo), gdesc(b_blk, COUT * 16), 1);
              }
            }
          }
          if constexpr (FMT != kFmtF16) {
            if constexpr (FMT == kFmtF16x2) {  // same registers, different shape: let the first group complete
              wg_commit();
              wg_wait<0>();
            }
#pragma unroll
            for (int g = 0; g < MT; ++g) acc_fence(acc[g]);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < Cfg::KS; ++ks) {
              const uint32_t b_blk = b_tap + (uint32_t)ks * Cfg::BLK;
              const uint32_t a_ks = a_tap + (uint32_t)(2 * ks * P + 1) * p.plane_stride;  // part 1: a_lo / [A8 | L8]
#pragma unroll
              for (int g = 0; g < MT; ++g) {
                if (g < ntiles) {
                  const uint32_t a = a_ks + (uint32_t)((g0 + g) * 64) * 16u;
                  if constexpr (FMT == kFmtF16x2)
                    wgmma_f16<COUT>(reinterpret_cast<float(&)[COUT / 2]>(acc[g]), gdesc(a, a_lbo), gdesc(b_blk, 2 * COUT * 16), 1);
                  else
                    wgmma_e4m3<COUT>(reinterpret_cast<float(&)[COUT / 2]>(acc[g][COUT / 2]), gdesc(a, a_lbo),
                                     gdesc(b_blk + 32 * COUT, COUT * 16));
                }
              }
            }
          }
          wg_commit();
#pragma unroll
          for (int g = 0; g < MT; ++g) acc_fence(acc[g]);
          if (!resident) {
            wg_wait<1>();  // the previous tap's products are done: its stage may be refilled
            if (prev_st >= 0 && leader) mbar_arrive(BAR(kBE + prev_st));
            prev_st = (int)st;
          }
        }
      }
      if (MODE == kConvT) epilogue(t);
    }
    if (MODE != kConvT) epilogue(0);
    if (MODE == kConvT && leader) mbar_arrive(BAR(kAE + (zz % kRing)));  // plane z-1 (unused) is done with
  }
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    CFB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (!p || q != cudaDriverEntryPointSuccess) throw std::runtime_error("cuTensorMapEncodeTiled unavailable");
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

// CP8 tensor (planes, Z, Y, X, 8 x fp16) as a 4-D TMA tensor map over 8-byte elements: the 16-byte voxel
// records of one x row are contiguous in memory, so (x, channel) is ONE inner dimension of 2*X elements and a
// box row is one contiguous run (box rows limited to 256 elements = 128 records).  Out-of-bounds elements are
// zero-filled: SAME padding at the patch border.
CUtensorMap make_map(const __half* base, int planes, Int3 sz, int bx, int by, int bplanes) {
  if (bx > 128) throw std::runtime_error("TMA box row limited to 128 voxel records");
  CUtensorMap m;
  cuuint64_t gdim[4] = {(cuuint64_t)sz.x * 2, (cuuint64_t)sz.y, (cuuint64_t)sz.z, (cuuint64_t)planes};
  cuuint64_t gstr[3] = {(cuuint64_t)sz.x * 16, (cuuint64_t)sz.x * sz.y * 16, (cuuint64_t)sz.x * sz.y * sz.z * 16};
  cuuint32_t box[4] = {(cuuint32_t)bx * 2, (cuuint32_t)by, 1, (cuuint32_t)bplanes};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, const_cast<__half*>(base), gdim, gstr, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return m;
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  return n;
}

template <int CIN, int COUT, int FMT, int MODE>
size_t smem_bytes(uint32_t slot_stride, int bstages) {
  using Cfg = ConvCfg<CIN, COUT, FMT>;
  return (size_t)kRing * slot_stride + kTailPad + (size_t)bstages * Cfg::TAP + stage_bytes<CIN, COUT, FMT, MODE>() + kBarBytes + 128;
}

// The cheapest feasible tiling of one layer by a static cost model: (halo amplification of the z-plane
// loads) / 2 + (M-tile positions per useful output), scaled by the wave quantisation of the grid, + a
// penalty for streamed (not resident) weights.  A grid of fewer columns than SMs is split along z into
// blocks of at least 2 output planes (each block reloads its two halo planes).
// Tests force the other code paths: CFB_FORCE_ZBLOCK=T (T output planes per CTA), CFB_FORCE_WEIGHT_RING=1
// (weights streamed through a 3-stage ring even where all taps would fit).  The row pitch is XT + 2, padded by junk columns
// where needed so that planes stay 128-byte aligned; fused pooling needs an even number of rows per tile.
template <int CIN, int COUT, int FMT, int MODE>
ConvTile choose_tile(int nb, Int3 sz) {
  using Cfg = ConvCfg<CIN, COUT, FMT>;
  constexpr int M = kConsumers * Cfg::MT * 64;  // positions per CTA
  std::vector<int> xts;
  for (int k = 1; k <= 32; ++k) {
    int xt = ceil_div(sz.x, k);
    xt += xt & 1;
    if (xt + 2 > 128 || (xt < 8 && k > 1)) continue;
    if (std::find(xts.begin(), xts.end(), xt) == xts.end()) xts.push_back(xt);
  }
  ConvTile best;
  best.cost = 1e30;
  const int ntaps = MODE == kConvT ? 4 : 27;
  // pass 0: pitch XT + 2 only; pass 1 (no aligned tiling exists, e.g. y extent 1): pitch padded with junk columns
  for (int pass = 0; pass < 2 && best.XT == 0; ++pass)
  for (int XT : xts) {
    for (int TY = std::min(16, sz.y); TY >= 1; --TY) {
      if (MODE == kConvPool && (TY & 1)) continue;
      int pitch = XT + 2;
      while (pass && ((TY + 2) * pitch) % 8) pitch += 2;
      if (((TY + 2) * pitch) % 8) continue;  // 128-byte planes: every TMA destination in a slot stays 128-byte aligned
      if (pitch > 128 || TY * pitch > M) continue;
      const uint32_t plane = (uint32_t)((TY + 2) * pitch * 16);
      const uint32_t slot = (uint32_t)(((size_t)Cfg::NPL * plane + 127) / 128 * 128);
      const size_t fixed = smem_bytes<CIN, COUT, FMT, MODE>(slot, 0);
      if (fixed >= (size_t)kMaxSmem) continue;
      int bs = (int)std::min<size_t>(((size_t)kMaxSmem - fixed) / Cfg::TAP, ntaps);
      if (bs < 2) continue;
      const int G = ceil_div(TY * pitch, 64);
      const double useful = (double)std::min(TY, sz.y) * std::min(XT, sz.x);
      const int ctas = nb * ceil_div(sz.x, XT) * ceil_div(sz.y, TY);
      const double waves = (double)ctas / sm_count();
      const double quant = std::ceil(waves) / waves;
      const double cost = (((double)(TY + 2) * pitch / useful) * 0.5 + ((double)G * 64 / useful)) * quant +
                          (bs == ntaps ? 0.0 : 0.1);
      if (cost < best.cost) {
        best.XT = XT; best.TY = TY; best.pitch = pitch; best.bstages = bs; best.resident = bs == ntaps; best.cost = cost;
      }
    }
  }
  if (best.XT == 0) throw std::runtime_error("conv3_wgmma: no tile configuration fits shared memory");
  const int cols = nb * ceil_div(sz.x, best.XT) * ceil_div(sz.y, best.TY);
  best.zblk = sz.z;
  if (cols < sm_count() && sz.z >= 4)
    best.zblk = std::max(2, ceil_div(sz.z, std::min(ceil_div(sm_count(), cols), sz.z / 2)));
  if (const char* f = getenv("CFB_FORCE_ZBLOCK")) best.zblk = std::max(1, std::min(atoi(f), sz.z));
  if (getenv("CFB_FORCE_WEIGHT_RING")) { best.bstages = std::min(best.bstages, 3); best.resident = false; }
  return best;
}

template <int CIN, int COUT, int FMT, int MODE>
void launch_cfg(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb,
                Int3 sz, bool relu, cudaStream_t s, const FusedTail* tail, __half* pool_out = nullptr) {
  using Cfg = ConvCfg<CIN, COUT, FMT>;
  const uint64_t key = ((uint64_t)sz.z << 48) ^ ((uint64_t)sz.y << 32) ^ ((uint64_t)sz.x << 16) ^ (uint64_t)nb;
  auto it = w.tuned->find(key);
  if (it == w.tuned->end()) it = w.tuned->emplace(key, choose_tile<CIN, COUT, FMT, MODE>(nb, sz)).first;
  const ConvTile& t = it->second;
  WgConvParams p{};
  p.Z = sz.z; p.Y = sz.y; p.X = sz.x;
  p.XT = t.XT; p.TY = t.TY; p.pitch = t.pitch;
  p.G = ceil_div(p.TY * p.pitch, 64);
  p.tiles_x = ceil_div(sz.x, p.XT);
  p.tiles_y = ceil_div(sz.y, p.TY);
  p.plane_stride = (uint32_t)((p.TY + 2) * p.pitch * 16);
  p.slot_stride = (uint32_t)((Cfg::NPL * (size_t)p.plane_stride + 127) / 128 * 128);
  p.planes_a = ca / 8; p.planes_b = cb / 8;
  p.wpacked = reinterpret_cast<const uint8_t*>(w.w); p.bias = w.bias; p.out = out; p.relu = relu ? 1 : 0;
  p.acc_scale = w.acc_scale;
  p.bstages = t.bstages; p.bresident = t.resident ? 1 : 0;
  p.zblk = t.zblk; p.zblocks = ceil_div(sz.z, t.zblk);
  p.out_pool = pool_out;
  const size_t smem = smem_bytes<CIN, COUT, FMT, MODE>(p.slot_stride, p.bstages);
  const CUtensorMap mapA = make_map(srcA, nb * p.planes_a * Cfg::P, sz, p.pitch, p.TY + 2, p.planes_a * Cfg::P);
  const CUtensorMap mapB = cb > 0 ? make_map(srcB, nb * p.planes_b * Cfg::P, sz, p.pitch, p.TY + 2, p.planes_b * Cfg::P) : mapA;
  const int grid = nb * p.tiles_x * p.tiles_y * p.zblocks;
  auto run = [&](auto kern) {
    CFB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kThreads, smem, s>>>(mapA, mapB, p);
    CFB_LAUNCH_CHECK();
  };
  if (tail) {
    if constexpr (CIN == 16 && COUT == 16 && MODE == kConv) {
      p.tail = *tail;
      run(conv3_wgmma_kernel<CIN, COUT, FMT, true, kConv>);
    } else {
      throw std::runtime_error("the fused head+blend tail needs a 16->16 layer");
    }
    return;
  }
  run(conv3_wgmma_kernel<CIN, COUT, FMT, false, MODE>);
}

template <int FMT>
void dispatch(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb, Int3 sz,
              bool relu, cudaStream_t s, const FusedTail* tail, __half* pool_out) {
  const int cin = ca + cb, cout = w.cout;
#define CFB_CASE(CI, CO) \
  if (cin == CI && cout == CO) return launch_cfg<CI, CO, FMT, kConv>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail);
  if (pool_out) {  // the two encoder layers that feed a pool
    if (cin == 16 && cout == 16) return launch_cfg<16, 16, FMT, kConvPool>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr, pool_out);
    if (cin == 32 && cout == 32) return launch_cfg<32, 32, FMT, kConvPool>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, nullptr, pool_out);
    throw std::runtime_error("conv3_wgmma: fused pooling exists for the 16->16 and 32->32 layers");
  }
  CFB_CASE(16, 16) CFB_CASE(16, 32) CFB_CASE(32, 32) CFB_CASE(32, 64) CFB_CASE(64, 64) CFB_CASE(64, 32) CFB_CASE(32, 16)
#undef CFB_CASE
  throw std::runtime_error("conv3_wgmma: unsupported channel configuration " + std::to_string(cin) + "->" + std::to_string(cout));
}

}  // namespace

void launch_conv3_wgmma(const __half* srcA, int ca, const __half* srcB, int cb, const PackedConv& w, __half* out, int nb,
                        Int3 sz, bool relu, cudaStream_t s, const ConvTail* tail, __half* pool_out) {
  if (ca % 16 || (cb % 16) || w.cin != ca + cb || w.taps != 27) throw std::runtime_error("conv3_wgmma: channel mismatch");
  if (pool_out && (tail || (sz.y & 1) || (sz.x & 1))) throw std::runtime_error("conv3_wgmma: pooling needs even y, x and no fused tail");
  FusedTail ft{};
  if (tail) {
    if (tail->channels > 8) throw std::runtime_error("fused tail: at most 8 channels");
    ft.head_w = tail->head_w; ft.head_b = tail->head_b; ft.patches = tail->patches; ft.mask = tail->mask; ft.out = tail->out;
    ft.channels = tail->channels; ft.op = tail->out_patch; ft.crop = tail->crop; ft.os = tail->out_size;
    ft.scale = tail->scale;
  }
  if (w.fmt == kFmtF16F8) dispatch<kFmtF16F8>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail ? &ft : nullptr, pool_out);
  else if (w.fmt == kFmtF16x2) dispatch<kFmtF16x2>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail ? &ft : nullptr, pool_out);
  else dispatch<kFmtF16>(srcA, ca, srcB, cb, w, out, nb, sz, relu, s, tail ? &ft : nullptr, pool_out);
}

void launch_convT_wgmma(const __half* in, const PackedConv& w, __half* out, int nb, Int3 in_size, cudaStream_t s) {
  if (w.taps != 4) throw std::runtime_error("convT_wgmma: weights are not a (1,2,2) transposed convolution");
#define CFB_CASE(CI, CO)                                                                                                   \
  if (w.cin == CI && w.cout == CO) {                                                                                       \
    if (w.fmt == kFmtF16F8) return launch_cfg<CI, CO, kFmtF16F8, kConvT>(in, CI, nullptr, 0, w, out, nb, in_size, false, s, nullptr); \
    if (w.fmt == kFmtF16x2) return launch_cfg<CI, CO, kFmtF16x2, kConvT>(in, CI, nullptr, 0, w, out, nb, in_size, false, s, nullptr); \
    return launch_cfg<CI, CO, kFmtF16, kConvT>(in, CI, nullptr, 0, w, out, nb, in_size, false, s, nullptr);                \
  }
  CFB_CASE(64, 32) CFB_CASE(32, 16)
#undef CFB_CASE
  throw std::runtime_error("convT_wgmma: unsupported channel configuration");
}

// ------------------------------------------------------------------------------------------
// Weight packing (host)
// ------------------------------------------------------------------------------------------
// power of two >= the largest |w| of a layer (f16f8 mode: beta = 2^14 / wmax', act_format.cuh)
static float weight_beta(const float* w, size_t n) {
  float wmax = 0.f;
  for (size_t i = 0; i < n; ++i) wmax = std::max(wmax, std::fabs(w[i]));
  if (!(wmax > 0.f) || !std::isfinite(wmax)) return 16384.0f;
  return 16384.0f / std::exp2(std::ceil(std::log2(wmax)));
}
static uint8_t to_e4m3(float v) { return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3); }

// One block per (tap, K step of 16 input channels), BLK = parts * 32 * cout bytes, rows are output channels,
// [chunk of 8 input channels][rows][16 bytes] (K-major core matrices):
//   f16   : [2][cout]      fp16(w)
//   f16x2 : [2][2 cout]    rows 0..cout-1 fp16(w), rows cout..2cout-1 fp16(w - fp16(w))
//   f16f8 : [2][cout] fp16(w beta), then [2][cout] x 16 e4m3: chunk 0 = WL8 = e4m3((w beta - WH) mu),
//           chunk 1 = W8 = e4m3(w delta) of the same 16 input channels
// `W(co, ci, tap)` reads the layer's fp32 weights; a transposed convolution has 4 taps (its output parities).
template <typename WF>
static void pack_blocks(WF W, const float* h_w, const float* h_bias, int cin, int cout, int taps, int fmt, PackedConv& out) {
  free_packed(out);
  const int parts = fmt_planes(fmt);
  const int KS = cin / 16;
  const size_t blk = (size_t)parts * 32 * cout;
  std::vector<uint8_t> buf((size_t)taps * KS * blk, 0);
  const float beta = fmt == kFmtF16F8 ? weight_beta(h_w, (size_t)cout * cin * taps) : 1.0f, delta = beta / kActLambda;
  auto put_half = [&](size_t off, float v) { const __half h = __float2half_rn(v); std::memcpy(&buf[off], &h, 2); };
  for (int t = 0; t < taps; ++t)
    for (int ks = 0; ks < KS; ++ks) {
      const size_t base = ((size_t)t * KS + ks) * blk;
      for (int kc = 0; kc < 2; ++kc)
        for (int co = 0; co < cout; ++co) {
          for (int e = 0; e < 8; ++e) {
            const int ci = ks * 16 + kc * 8 + e;
            const float wv = W(co, ci, t);
            if (fmt == kFmtF16) {
              put_half(base + ((size_t)kc * cout + co) * 16 + 2 * e, wv);
            } else if (fmt == kFmtF16x2) {
              const float hi = __half2float(__float2half_rn(wv));
              put_half(base + ((size_t)kc * 2 * cout + co) * 16 + 2 * e, wv);
              put_half(base + ((size_t)kc * 2 * cout + cout + co) * 16 + 2 * e, wv - hi);
            } else {
              put_half(base + ((size_t)kc * cout + co) * 16 + 2 * e, wv * beta);
            }
          }
          if (fmt == kFmtF16F8) {
            uint8_t* dst = &buf[base + (size_t)32 * cout + ((size_t)kc * cout + co) * 16];
            for (int j = 0; j < 16; ++j) {
              const float w0 = W(co, ks * 16 + j, t), wb = w0 * beta;
              dst[j] = kc ? to_e4m3(w0 * delta) : to_e4m3((wb - __half2float(__float2half_rn(wb))) * kWgtMu);
            }
          }
        }
    }
  out.cin = cin; out.cout = cout; out.parts = parts; out.fmt = fmt; out.taps = taps;
  out.acc_scale = fmt == kFmtF16F8 ? 1.0f / (kActAlpha * beta) : 1.0f;
  out.tuned = std::make_shared<std::map<uint64_t, ConvTile>>();
  out.bytes = buf.size();
  CFB_CUDA(cudaMalloc(&out.w, out.bytes));
  CFB_CUDA(cudaMemcpy(out.w, buf.data(), out.bytes, cudaMemcpyHostToDevice));
  CFB_CUDA(cudaMalloc(&out.bias, cout * sizeof(float)));
  CFB_CUDA(cudaMemcpy(out.bias, h_bias, cout * sizeof(float), cudaMemcpyHostToDevice));
}

void pack_conv3_weights(const float* h_w, const float* h_bias, int cin, int cout, int fmt, PackedConv& out) {
  pack_blocks([&](int co, int ci, int t) { return h_w[((size_t)co * cin + ci) * 27 + t]; }, h_w, h_bias, cin, cout, 27, fmt, out);
}

// h_w: (cin, cout, 1, 2, 2); tap = (oy & 1) * 2 + (ox & 1)
void pack_convT_weights(const float* h_w, const float* h_bias, int cin, int cout, int fmt, PackedConv& out) {
  pack_blocks([&](int co, int ci, int t) { return h_w[((size_t)ci * cout + co) * 4 + t]; }, h_w, h_bias, cin, cout, 4, fmt, out);
}

void free_packed(PackedConv& p) {
  if (p.w) cudaFree(p.w);
  if (p.bias) cudaFree(p.bias);
  p = PackedConv{};
}

}  // namespace cfb
