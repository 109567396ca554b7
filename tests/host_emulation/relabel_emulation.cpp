// TEST INFRASTRUCTURE: runs the device code of chunkflow_b200/csrc/label_table.cuh on the host, one "thread" in a one-lane
// warp (grid 1 x 1, so every grid-stride loop walks the whole range; a "warp" holds the 2, 4 or 16 ids of one 16-byte load, so
// runs are combined inside a lane but never across lanes; atomics are plain read-modify-writes), so that the LOGIC of the
// count, plan and apply kernels is compared with oracle/relabel_oracle.py on machines without a GPU
// (tests/test_relabel_oracle.py builds this file with g++).  The block scan between lt_block_count_kernel and lt_rank_kernel
// (cc_scan_blocks_kernel, a 1024-thread kernel) is replaced by a serial exclusive scan here.  Concurrency and runs that span
// lanes are what the `-m gpu` tests add.
#include <algorithm>
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
struct uint4 { uint32_t x, y, z, w; };
template <typename T> static T atomicCAS(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }
template <typename T> static T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <typename T> static T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <typename T> static T atomicMin(T* p, T v) { T o = *p; *p = std::min(o, v); return o; }
template <typename T> static T atomicMax(T* p, T v) { T o = *p; *p = std::max(o, v); return o; }
template <typename T> static T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
static void __threadfence() {}
static int __ffs(int v) { return __builtin_ffs(v); }
static int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static int __popc(uint32_t v) { return __builtin_popcount(v); }

// a one-lane warp
#define EV_WARP 1
static int ev_lane() { return 0; }
static unsigned long long ev_shfl_up(unsigned long long v) { return v; }
static uint32_t ev_ballot(bool p) { return p ? 1u : 0u; }
static unsigned long long ev_warp_sum(unsigned long long v) { return v; }

constexpr int kT = 256;
#include "../../chunkflow_b200/csrc/label_table.cuh"

template <typename TI>
static void run_apply(const void* in, int64_t n, const LtTable& t, void* out, bool wide) {
  if (wide) lt_apply_kernel<TI, uint64_t>((const TI*)in, n, t, (uint64_t*)out);
  else lt_apply_kernel<TI, TI>((const TI*)in, n, t, (TI*)out);
}

// labels: n ids of 1, 4 or 8 bytes.  Builds the table (sorted by id into h_ids / h_counts / h_first, capacity `slots`), plans
// (dust when use_dust, keep-list when num_keep >= 0, ranks when renumber) and applies into `out` (uint64 when renumber, else
// the input's width; may be `labels` itself).  info = {entries failing the dust test, surviving non-zero ids, new maximum}.
// -> number of labels, -1 when the table overflowed, -2 when apply met an id the table does not hold
extern "C" int64_t emu_relabel(const void* labels, int bytes, int64_t n, int64_t slots, int use_dust, int64_t dust_threshold,
                               const uint64_t* keep, int64_t num_keep, int renumber, uint64_t base_id, uint64_t* h_ids,
                               uint32_t* h_counts, uint32_t* h_first, void* out, uint64_t* info) {
  std::vector<unsigned long long> stats(kLtStatWords, 0), wide(2 * slots, 0);
  std::vector<uint32_t> words(4 * slots, 0);
  LtTable t;
  t.stats = stats.data();
  t.keys = wide.data(); t.newval = t.keys + slots;
  t.state = words.data(); t.count = t.state + slots; t.first = t.count + slots; t.flags = t.first + slots;
  std::fill(t.first, t.first + slots, 0xFFFFFFFFu);
  t.mask = (unsigned long long)(slots - 1);
  if (bytes == 1) lt_count_kernel<uint8_t>((const uint8_t*)labels, n, t);
  else if (bytes == 4) lt_count_kernel<uint32_t>((const uint32_t*)labels, n, t);
  else if (bytes == 8) lt_count_kernel<uint64_t>((const uint64_t*)labels, n, t);
  else return -3;
  if (stats[kLtOverflow]) return -1;
  std::vector<uint32_t> order;
  for (int64_t i = 0; i < slots; ++i)
    if (t.state[i] == 2u) order.push_back((uint32_t)i);
  if ((int64_t)order.size() != (int64_t)stats[kLtLabels]) return -4;
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return t.keys[a] < t.keys[b]; });
  for (size_t i = 0; i < order.size(); ++i) { h_ids[i] = t.keys[order[i]]; h_counts[i] = t.count[order[i]]; h_first[i] = t.first[order[i]]; }

  const int64_t nblocks = ((n + 31) / 32 + kLtBlockWords - 1) / kLtBlockWords;
  std::vector<uint32_t> bits(nblocks * kLtBlockWords, 0), block_count(nblocks, 0);
  if (num_keep > 0) lt_keep_kernel((const unsigned long long*)keep, num_keep, t);
  lt_decide_kernel(t, use_dust, (long long)dust_threshold, num_keep >= 0, renumber, bits.data());
  if (renumber) {
    lt_block_count_kernel(bits.data(), nblocks, block_count.data());
    uint32_t run = 0;
    for (auto& c : block_count) { const uint32_t v = c; c = run; run += v; }
    if (run != stats[kLtSurvivors]) return -5;
    lt_rank_kernel(t, bits.data(), block_count.data(), (unsigned long long)base_id);
  }
  info[0] = stats[kLtDust];
  info[1] = stats[kLtSurvivors];
  info[2] = renumber ? (stats[kLtSurvivors] ? stats[kLtSurvivors] + base_id : 0) : stats[kLtMax];
  if (bytes == 1) run_apply<uint8_t>(labels, n, t, out, renumber);
  else if (bytes == 4) run_apply<uint32_t>(labels, n, t, out, renumber);
  else run_apply<uint64_t>(labels, n, t, out, renumber);
  if (stats[kLtMissing]) return -2;
  return (int64_t)stats[kLtLabels];
}
