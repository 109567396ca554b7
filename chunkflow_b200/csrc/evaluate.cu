// `evaluate-segmentation` on the device (DESIGN.md section 0, row f5): Segmentation.evaluate (reference chunk/segmentation.py:33-67)
// -> the gala metrics (reference lib/gala/evaluate.py), restated in oracle/evaluation_oracle.py.  One pass over the two label
// volumes builds the sparse contingency table; everything the five scores need follows from the table (evaluate_kernels.cuh),
// and the scores themselves from a handful of exact statistics on the host (evaluate_scores.h).
//
// Wide ids: the table is keyed by the two 64-bit ids themselves (a 128-bit key).  The alternative, a first pass that maps
// every id to a dense one, reads both volumes twice and writes a uint32 volume per side; the 128-bit key reads each voxel's
// ids once, and its only cost is 8 more bytes per table slot (tools/bench_evaluate.py counts both kinds of traffic).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"
#include "evaluate_scores.h"

namespace cfb {
namespace {

constexpr int kT = 256;

#include "evaluate_kernels.cuh"

int ev_grid(int64_t items) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(items, kT), 132 * 16));
}

void ev_check_slots(int64_t table_slots) {
  if (table_slots < 32 || (table_slots & (table_slots - 1)) || table_slots >= ((int64_t)1 << 31))
    throw std::invalid_argument("evaluate: table_slots must be a power of two in [32, 2^31)");
}

// workspace: stats (kEvStatWords x 8 B) | pair seg ids | pair gt ids | row ids | col ids (8 B per slot each) |
//            pair state | pair count | row state | row all | row nz | col state | col all | col nz (4 B per slot each)
EvTables ev_tables(void* d_workspace, int64_t slots) {
  EvTables t;
  t.stats = static_cast<unsigned long long*>(d_workspace);
  t.pk1 = t.stats + kEvStatWords;
  t.pk2 = t.pk1 + slots;
  t.rkey = t.pk2 + slots;
  t.ckey = t.rkey + slots;
  uint32_t* u = reinterpret_cast<uint32_t*>(t.ckey + slots);
  t.pstate = u; t.pcount = u + slots;
  t.rstate = u + 2 * slots; t.rall = u + 3 * slots; t.rnz = u + 4 * slots;
  t.cstate = u + 5 * slots; t.call = u + 6 * slots; t.cnz = u + 7 * slots;
  t.mask = (unsigned long long)(slots - 1);
  return t;
}

template <typename TS>
void ev_launch_pairs(const TS* seg, const void* gt, int32_t gt_dtype, int64_t n, const EvTables& t, cudaStream_t s) {
  const int grid = ev_grid(n);
  if (gt_dtype == CFB_DTYPE_U8) ev_pairs_kernel<TS, uint8_t><<<grid, kT, 0, s>>>(seg, (const uint8_t*)gt, n, t);
  else if (gt_dtype == CFB_DTYPE_U32) ev_pairs_kernel<TS, uint32_t><<<grid, kT, 0, s>>>(seg, (const uint32_t*)gt, n, t);
  else if (gt_dtype == CFB_DTYPE_U64) ev_pairs_kernel<TS, uint64_t><<<grid, kT, 0, s>>>(seg, (const uint64_t*)gt, n, t);
  else throw std::invalid_argument("evaluate: ground-truth dtype must be uint8, uint32 or uint64");
  CFB_LAUNCH_CHECK();
}

template <typename F>
int guarded_eval(F&& f) {
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

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int64_t cfb_evaluate_workspace(int64_t table_slots) {
  if (table_slots <= 0) return 0;
  return kEvStatWords * 8 + table_slots * (4 * 8 + 8 * 4);
}

extern "C" int cfb_contingency_device(const void* d_seg, int32_t seg_dtype, const void* d_gt, int32_t gt_dtype, int64_t z, int64_t y,
                                      int64_t x, void* d_workspace, int64_t table_slots, int64_t* num_pairs, void* stream) {
  return guarded_eval([&]() -> int {
    if (!d_seg || !d_gt || !d_workspace || !num_pairs) throw std::invalid_argument("evaluate: null argument");
    if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX) throw std::invalid_argument("evaluate: bad volume size");
    const int64_t n = z * y * x;
    if (n >= (int64_t)UINT32_MAX) throw std::invalid_argument("evaluate: more than 2^32 - 1 voxels");
    ev_check_slots(table_slots);
    cudaStream_t s = (cudaStream_t)stream;
    const EvTables t = ev_tables(d_workspace, table_slots);
    CFB_CUDA(cudaMemsetAsync(t.stats, 0, kEvStatWords * 8, s));
    CFB_CUDA(cudaMemsetAsync(t.pstate, 0, (size_t)table_slots * 8 * 4, s));   // all states and counts
    if (seg_dtype == CFB_DTYPE_U8) ev_launch_pairs((const uint8_t*)d_seg, d_gt, gt_dtype, n, t, s);
    else if (seg_dtype == CFB_DTYPE_U32) ev_launch_pairs((const uint32_t*)d_seg, d_gt, gt_dtype, n, t, s);
    else if (seg_dtype == CFB_DTYPE_U64) ev_launch_pairs((const uint64_t*)d_seg, d_gt, gt_dtype, n, t, s);
    else throw std::invalid_argument("evaluate: segmentation dtype must be uint8, uint32 or uint64");
    ev_margins_kernel<<<ev_grid(table_slots), kT, 0, s>>>(t);
    CFB_LAUNCH_CHECK();
    ev_side_kernel<<<ev_grid(table_slots), kT, 0, s>>>(t.rstate, t.rall, t.rnz, table_slots, t.stats + kEvS2, t.stats + kEvXlR);
    CFB_LAUNCH_CHECK();
    ev_side_kernel<<<ev_grid(table_slots), kT, 0, s>>>(t.cstate, t.call, t.cnz, table_slots, t.stats + kEvS3, t.stats + kEvXlS);
    CFB_LAUNCH_CHECK();
    unsigned long long h[kEvStatWords];
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_pairs = (int64_t)h[kEvPairs];
    if (h[kEvOverflow]) {
      set_last_error("evaluate: the contingency table is too small for this many label pairs");
      return CFB_ERR_CAPACITY;
    }
    if (h[kEvN] != (unsigned long long)n) throw std::runtime_error("evaluate: the contingency table does not add up to the voxel count");
    return CFB_OK;
  });
}

extern "C" int cfb_contingency_scores(void* d_workspace, int64_t table_slots, double size_threshold, cfb_seg_scores* out, void* stream) {
  return guarded_eval([&]() -> int {
    if (!d_workspace || !out) throw std::invalid_argument("evaluate scores: null argument");
    if (out->struct_size != (int32_t)sizeof(cfb_seg_scores)) throw std::invalid_argument("evaluate scores: cfb_seg_scores size mismatch");
    ev_check_slots(table_slots);
    cudaStream_t s = (cudaStream_t)stream;
    const EvTables t = ev_tables(d_workspace, table_slots);
    CFB_CUDA(cudaMemsetAsync(t.stats + kEvK, 0, 8, s));
    ev_threshold_kernel<<<ev_grid(table_slots), kT, 0, s>>>(t, size_threshold);
    CFB_LAUNCH_CHECK();
    unsigned long long h[kEvStatWords];
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (h[kEvOverflow]) throw std::invalid_argument("evaluate scores: the table in the workspace is incomplete (it overflowed)");
    const int32_t size = out->struct_size;
    std::memset(out, 0, sizeof(*out));
    out->struct_size = size;
    out->n = h[kEvN];
    out->sum_sq_pairs = h[kEvS1];
    out->sum_sq_rows = h[kEvS2];
    out->sum_sq_cols = h[kEvS3];
    out->n_both_nonzero = h[kEvNBoth];
    out->seg_ids = h[kEvSegIds];
    out->gt_ids = h[kEvGtIds];
    out->pairs = h[kEvPairs];
    out->pairs_over_threshold = h[kEvK];
    out->size_threshold = size_threshold;
    out->xlog_pairs = ev_compose_xlog(h + kEvXlC);
    out->xlog_rows = ev_compose_xlog(h + kEvXlR);
    out->xlog_cols = ev_compose_xlog(h + kEvXlS);
    ev_scores(out);
    return CFB_OK;
  });
}

extern "C" int cfb_contingency_read(void* d_workspace, int64_t table_slots, int64_t num_pairs, uint64_t* h_seg, uint64_t* h_gt,
                                    uint32_t* h_count, void* stream) {
  return guarded_eval([&]() -> int {
    if (!d_workspace || num_pairs < 0 || num_pairs > table_slots) throw std::invalid_argument("evaluate read: bad argument");
    ev_check_slots(table_slots);
    if (num_pairs == 0) return CFB_OK;
    if (!h_seg || !h_gt || !h_count) throw std::invalid_argument("evaluate read: null output");
    cudaStream_t s = (cudaStream_t)stream;
    const EvTables t = ev_tables(d_workspace, table_slots);
    std::vector<unsigned long long> k1((size_t)table_slots), k2((size_t)table_slots);
    std::vector<uint32_t> st((size_t)table_slots), ct((size_t)table_slots);
    CFB_CUDA(cudaMemcpyAsync(k1.data(), t.pk1, (size_t)table_slots * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(k2.data(), t.pk2, (size_t)table_slots * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(st.data(), t.pstate, (size_t)table_slots * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(ct.data(), t.pcount, (size_t)table_slots * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> order;
    order.reserve((size_t)num_pairs);
    for (int64_t i = 0; i < table_slots; ++i)
      if (st[i] == 2u) order.push_back((uint32_t)i);
    if ((int64_t)order.size() != num_pairs) throw std::invalid_argument("evaluate read: num_pairs does not match the table");
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return k1[a] != k1[b] ? k1[a] < k1[b] : k2[a] < k2[b]; });
    for (size_t i = 0; i < order.size(); ++i) {
      h_seg[i] = k1[order[i]];
      h_gt[i] = k2[order[i]];
      h_count[i] = ct[order[i]];
    }
    return CFB_OK;
  });
}
