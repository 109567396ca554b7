// TEST INFRASTRUCTURE: runs the device code of chunkflow_b200/csrc/evaluate_kernels.cuh on the host, one "thread" in a
// one-lane warp (grid 1 x 1, so every grid-stride loop walks the whole range and every run of equal pairs has length 1;
// atomics are plain read-modify-writes), so that the LOGIC of the contingency-table kernels and of the host scoring code
// (csrc/evaluate_scores.h) is compared with oracle/evaluation_oracle.py on machines without a GPU
// (tests/test_evaluate_oracle.py builds this file with g++).  Concurrency and run aggregation are what the `-m gpu` tests add.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
struct EmuDim { unsigned x = 0; };
static EmuDim blockIdx, threadIdx;
static struct { unsigned x = 1; } blockDim, gridDim;
template <typename T> static T atomicCAS(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }
template <typename T> static T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <typename T> static T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
static void __threadfence() {}
static int __ffs(int v) { return __builtin_ffs(v); }

// a one-lane warp
#define EV_WARP 1
static int ev_lane() { return 0; }
static unsigned long long ev_shfl_up(unsigned long long v) { return v; }
static uint32_t ev_ballot(bool p) { return p ? 1u : 0u; }
static unsigned long long ev_warp_sum(unsigned long long v) { return v; }

constexpr int kT = 256;
#include "../../chunkflow_b200/csrc/evaluate_kernels.cuh"
#include "../../chunkflow_b200/csrc/evaluate_scores.h"

template <typename TS, typename TG>
static void run_pairs(const void* seg, const void* gt, int64_t n, const EvTables& t) {
  ev_pairs_kernel<TS, TG>((const TS*)seg, (const TG*)gt, n, t);
}

template <typename TS>
static int dispatch_gt(const void* seg, const void* gt, int gt_bytes, int64_t n, const EvTables& t) {
  if (gt_bytes == 1) run_pairs<TS, uint8_t>(seg, gt, n, t);
  else if (gt_bytes == 4) run_pairs<TS, uint32_t>(seg, gt, n, t);
  else if (gt_bytes == 8) run_pairs<TS, uint64_t>(seg, gt, n, t);
  else return -3;
  return 0;
}

// seg / gt: n labels of 1, 4 or 8 bytes.  -> number of pairs (triples sorted by (seg, gt) into the outputs, capacity
// `slots`, and the statistics + scores of `size_threshold` into *out), -1 when a table overflowed
extern "C" int64_t emu_evaluate(const void* seg, int seg_bytes, const void* gt, int gt_bytes, int64_t n, int64_t slots, double size_threshold,
                                uint64_t* h_seg, uint64_t* h_gt, uint32_t* h_count, cfb_seg_scores* out) {
  std::vector<unsigned long long> stats(kEvStatWords, 0), keys(4 * slots, 0);
  std::vector<uint32_t> words(8 * slots, 0);
  EvTables t;
  t.stats = stats.data();
  t.pk1 = keys.data(); t.pk2 = t.pk1 + slots; t.rkey = t.pk2 + slots; t.ckey = t.rkey + slots;
  uint32_t* u = words.data();
  t.pstate = u; t.pcount = u + slots; t.rstate = u + 2 * slots; t.rall = u + 3 * slots; t.rnz = u + 4 * slots;
  t.cstate = u + 5 * slots; t.call = u + 6 * slots; t.cnz = u + 7 * slots;
  t.mask = (unsigned long long)(slots - 1);
  int rc;
  if (seg_bytes == 1) rc = dispatch_gt<uint8_t>(seg, gt, gt_bytes, n, t);
  else if (seg_bytes == 4) rc = dispatch_gt<uint32_t>(seg, gt, gt_bytes, n, t);
  else if (seg_bytes == 8) rc = dispatch_gt<uint64_t>(seg, gt, gt_bytes, n, t);
  else rc = -3;
  if (rc) return rc;
  ev_margins_kernel(t);
  ev_side_kernel(t.rstate, t.rall, t.rnz, slots, t.stats + kEvS2, t.stats + kEvXlR);
  ev_side_kernel(t.cstate, t.call, t.cnz, slots, t.stats + kEvS3, t.stats + kEvXlS);
  if (stats[kEvOverflow]) return -1;
  ev_threshold_kernel(t, size_threshold);
  std::vector<uint32_t> order;
  for (int64_t i = 0; i < slots; ++i)
    if (t.pstate[i] == 2u) order.push_back((uint32_t)i);
  if ((int64_t)order.size() != (int64_t)stats[kEvPairs]) return -2;
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return t.pk1[a] != t.pk1[b] ? t.pk1[a] < t.pk1[b] : t.pk2[a] < t.pk2[b]; });
  for (size_t i = 0; i < order.size(); ++i) { h_seg[i] = t.pk1[order[i]]; h_gt[i] = t.pk2[order[i]]; h_count[i] = t.pcount[order[i]]; }
  std::memset(out, 0, sizeof(*out));
  out->struct_size = (int32_t)sizeof(*out);
  out->n = stats[kEvN]; out->sum_sq_pairs = stats[kEvS1]; out->sum_sq_rows = stats[kEvS2]; out->sum_sq_cols = stats[kEvS3];
  out->n_both_nonzero = stats[kEvNBoth]; out->seg_ids = stats[kEvSegIds]; out->gt_ids = stats[kEvGtIds];
  out->pairs = stats[kEvPairs]; out->pairs_over_threshold = stats[kEvK]; out->size_threshold = size_threshold;
  out->xlog_pairs = ev_compose_xlog(t.stats + kEvXlC);
  out->xlog_rows = ev_compose_xlog(t.stats + kEvXlR);
  out->xlog_cols = ev_compose_xlog(t.stats + kEvXlS);
  ev_scores(out);
  return (int64_t)stats[kEvPairs];
}

extern "C" int emu_scores_size() { return (int)sizeof(cfb_seg_scores); }
