// Segmentation clean-up on the device (DESIGN.md section 0, row f6): what the reference's Segmentation does with fastremap
// (reference chunk/segmentation.py: remap :69-84, mask_fragments :86-90, mask_except :92-109; `mask-out-objects`,
// flow/flow.py:2015-2050), restated in oracle/relabel_oracle.py.  The volume is read once to build the table of its labels
// (count pass), every entry's new value is planned from the table alone, and the volume is read a second time and written once
// (apply pass): dust removal, a keep-list and renumbering share these two reads however they are combined.  label_table.cuh
// holds the kernels; the raster-order ranking of `remap` uses the block scan of `connected-components` (raster_scan.cuh).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "chunkflow_b200.h"
#include "common.cuh"

namespace cfb {
namespace {

constexpr int kT = 256;

#include "label_table.cuh"
#include "raster_scan.cuh"

int lt_grid(int64_t items) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(items, kT), 132 * 16));
}

void lt_check_slots(int64_t table_slots) {
  if (table_slots < 32 || (table_slots & (table_slots - 1)) || table_slots >= ((int64_t)1 << 31))
    throw std::invalid_argument("label table: table_slots must be a power of two in [32, 2^31)");
}

void lt_check_voxels(int64_t n) {
  if (n <= 0) throw std::invalid_argument("label table: bad volume size");
  if (n >= (int64_t)UINT32_MAX) throw std::invalid_argument("label table: more than 2^32 - 2 voxels");
}

int lt_dtype_bytes(int32_t dtype) {
  if (dtype == CFB_DTYPE_U8) return 1;
  if (dtype == CFB_DTYPE_U32) return 4;
  if (dtype == CFB_DTYPE_U64) return 8;
  throw std::invalid_argument("label table: label dtype must be uint8, uint32 or uint64");
}

int64_t lt_scan_blocks(int64_t n) { return ceil_div64(ceil_div64(n, 32), kLtBlockWords); }

// workspace: stats (kLtStatWords x 8 B) | ids | new values (8 B per slot each) | state | count | first | flags (4 B per slot
//            each) | first-voxel flags (one bit per voxel, whole scan blocks) | block counts | total (4 B each)
LtTable lt_table(void* d_workspace, int64_t slots) {
  LtTable t;
  t.stats = static_cast<unsigned long long*>(d_workspace);
  t.keys = t.stats + kLtStatWords;
  t.newval = t.keys + slots;
  uint32_t* u = reinterpret_cast<uint32_t*>(t.newval + slots);
  t.state = u; t.count = u + slots; t.first = u + 2 * slots; t.flags = u + 3 * slots;
  t.mask = (unsigned long long)(slots - 1);
  return t;
}

template <typename TI>
void lt_launch_apply(const TI* in, int64_t n, const LtTable& t, void* out, int32_t out_dtype, cudaStream_t s) {
  const int grid = lt_grid(ceil_div64(n, 16 / (int64_t)sizeof(TI)));
  if (out_dtype == CFB_DTYPE_U64) launch(lt_apply_kernel<TI, uint64_t>, grid, kT, 0, s, in, n, t, (uint64_t*)out);
  else launch(lt_apply_kernel<TI, TI>, grid, kT, 0, s, in, n, t, (TI*)out);
}

}  // namespace
}  // namespace cfb

using namespace cfb;

extern "C" int64_t cfb_label_table_workspace(int64_t voxels, int64_t table_slots) {
  if (voxels <= 0 || table_slots <= 0) return 0;
  const int64_t nblocks = lt_scan_blocks(voxels);
  return kLtStatWords * 8 + table_slots * (2 * 8 + 4 * 4) + (nblocks * kLtBlockWords + nblocks + 1) * 4;
}

extern "C" int cfb_label_table_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, void* d_workspace,
                                      int64_t table_slots, int64_t* num_labels, void* stream) {
  return guarded([&]() -> int {
    if (!d_labels || !d_workspace || !num_labels) throw std::invalid_argument("label table: null argument");
    if (z <= 0 || y <= 0 || x <= 0 || z > INT32_MAX || y > INT32_MAX || x > INT32_MAX) throw std::invalid_argument("label table: bad volume size");
    const int64_t n = z * y * x;
    lt_check_voxels(n);
    lt_check_slots(table_slots);
    if ((uintptr_t)d_labels % 16) throw std::invalid_argument("label table: the volume must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    const LtTable t = lt_table(d_workspace, table_slots);
    CFB_CUDA(cudaMemsetAsync(t.stats, 0, kLtStatWords * 8, s));
    CFB_CUDA(cudaMemsetAsync(t.state, 0, (size_t)table_slots * 2 * 4, s));      // states and counts
    CFB_CUDA(cudaMemsetAsync(t.first, 0xFF, (size_t)table_slots * 4, s));       // atomicMin target
    const int grid = lt_grid(ceil_div64(n, 16 / lt_dtype_bytes(dtype)));
    if (dtype == CFB_DTYPE_U8) launch(lt_count_kernel<uint8_t>, grid, kT, 0, s, (const uint8_t*)d_labels, n, t);
    else if (dtype == CFB_DTYPE_U32) launch(lt_count_kernel<uint32_t>, grid, kT, 0, s, (const uint32_t*)d_labels, n, t);
    else launch(lt_count_kernel<uint64_t>, grid, kT, 0, s, (const uint64_t*)d_labels, n, t);
    unsigned long long h[kLtStatWords];
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    *num_labels = (int64_t)h[kLtLabels];
    if (h[kLtOverflow]) {
      set_last_error("label table: the table is too small for this many labels");
      return CFB_ERR_CAPACITY;
    }
    return CFB_OK;
  });
}

extern "C" int cfb_label_table_read(void* d_workspace, int64_t table_slots, int64_t num_labels, uint64_t* h_ids, uint32_t* h_counts,
                                    uint32_t* h_first, void* stream) {
  return guarded([&]() -> int {
    if (!d_workspace || num_labels < 0 || num_labels > table_slots) throw std::invalid_argument("label table read: bad argument");
    lt_check_slots(table_slots);
    if (num_labels == 0) return CFB_OK;
    if (!h_ids || !h_counts || !h_first) throw std::invalid_argument("label table read: null output");
    cudaStream_t s = (cudaStream_t)stream;
    const LtTable t = lt_table(d_workspace, table_slots);
    std::vector<unsigned long long> keys((size_t)table_slots);
    std::vector<uint32_t> words((size_t)table_slots * 3);   // state | count | first
    CFB_CUDA(cudaMemcpyAsync(keys.data(), t.keys, (size_t)table_slots * 8, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaMemcpyAsync(words.data(), t.state, (size_t)table_slots * 3 * 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    const uint32_t *st = words.data(), *ct = st + table_slots, *ft = ct + table_slots;
    std::vector<uint32_t> order;
    order.reserve((size_t)num_labels);
    for (int64_t i = 0; i < table_slots; ++i)
      if (st[i] == 2u) order.push_back((uint32_t)i);
    if ((int64_t)order.size() != num_labels) throw std::invalid_argument("label table read: num_labels does not match the table");
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
    for (size_t i = 0; i < order.size(); ++i) {
      h_ids[i] = keys[order[i]];
      h_counts[i] = ct[order[i]];
      h_first[i] = ft[order[i]];
    }
    return CFB_OK;
  });
}

extern "C" int cfb_label_table_plan(void* d_workspace, int64_t table_slots, int64_t voxels, int32_t use_dust, int64_t dust_threshold,
                                    const uint64_t* d_keep_ids, int64_t num_keep, int32_t renumber, uint64_t base_id,
                                    int64_t* num_dust, int64_t* num_survivors, uint64_t* new_max, void* stream) {
  return guarded([&]() -> int {
    if (!d_workspace) throw std::invalid_argument("label plan: null workspace");
    lt_check_voxels(voxels);
    lt_check_slots(table_slots);
    if (num_keep > 0 && !d_keep_ids) throw std::invalid_argument("label plan: null keep-list");
    const bool use_keep = num_keep >= 0;   // an empty keep-list masks everything; a negative count means "no keep-list"
    cudaStream_t s = (cudaStream_t)stream;
    const LtTable t = lt_table(d_workspace, table_slots);
    const int64_t nblocks = lt_scan_blocks(voxels);
    uint32_t* bits = t.flags + table_slots;
    uint32_t* block_count = bits + nblocks * kLtBlockWords;
    uint32_t* d_total = block_count + nblocks;
    unsigned long long h[kLtStatWords];
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (h[kLtOverflow]) throw std::invalid_argument("label plan: the table in the workspace is incomplete (it overflowed)");
    CFB_CUDA(cudaMemsetAsync(t.stats + kLtDust, 0, (kLtStatWords - kLtDust) * 8, s));
    CFB_CUDA(cudaMemsetAsync(t.flags, 0, (size_t)table_slots * 4, s));
    if (renumber) CFB_CUDA(cudaMemsetAsync(bits, 0, (size_t)nblocks * kLtBlockWords * 4, s));
    if (num_keep > 0) launch(lt_keep_kernel, lt_grid(num_keep), kT, 0, s, (const unsigned long long*)d_keep_ids, num_keep, t);
    launch(lt_decide_kernel, lt_grid(table_slots), kT, 0, s, t, use_dust ? 1 : 0, (long long)dust_threshold, use_keep ? 1 : 0,
           renumber ? 1 : 0, bits);
    if (renumber) {
      launch(lt_block_count_kernel, lt_grid(nblocks * EV_WARP), kT, 0, s, bits, nblocks, block_count);
      launch(cc_scan_blocks_kernel, 1, 1024, 0, s, block_count, nblocks, d_total);
      launch(lt_rank_kernel, lt_grid(table_slots), kT, 0, s, t, bits, block_count, (unsigned long long)base_id);
    }
    uint32_t total = 0;
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    if (renumber) CFB_CUDA(cudaMemcpyAsync(&total, d_total, 4, cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    const unsigned long long survivors = h[kLtSurvivors];
    if (renumber) {
      if ((unsigned long long)total != survivors) throw std::runtime_error("label plan: the first voxels of the surviving labels are not distinct");
      if (survivors > UINT64_MAX - base_id) throw std::invalid_argument("label plan: base_id + number of labels exceeds 2^64 - 1");
    }
    const unsigned long long done[2] = {renumber ? 1ULL : 0ULL, 1ULL};   // kLtRenumbered, kLtPlanned: the new values may be applied
    CFB_CUDA(cudaMemcpyAsync(t.stats + kLtRenumbered, done, sizeof(done), cudaMemcpyHostToDevice, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (num_dust) *num_dust = (int64_t)h[kLtDust];
    if (num_survivors) *num_survivors = (int64_t)survivors;
    // the maximum of the relabelled volume: 0 when nothing non-zero survives, whatever base_id (reference segmentation.py:81-83)
    if (new_max) *new_max = renumber ? (survivors ? survivors + base_id : 0ULL) : h[kLtMax];
    return CFB_OK;
  });
}

extern "C" int cfb_label_apply_device(const void* d_in, int32_t in_dtype, int64_t voxels, void* d_workspace, int64_t table_slots,
                                      void* d_out, int32_t out_dtype, void* stream) {
  return guarded([&]() -> int {
    if (!d_in || !d_workspace || !d_out) throw std::invalid_argument("label apply: null argument");
    lt_check_voxels(voxels);
    lt_check_slots(table_slots);
    const int in_bytes = lt_dtype_bytes(in_dtype);
    if (out_dtype != in_dtype && out_dtype != CFB_DTYPE_U64) throw std::invalid_argument("label apply: the output is of the input's dtype or uint64");
    if (d_out == d_in && out_dtype != in_dtype) throw std::invalid_argument("label apply: in place needs equal dtypes");
    if ((uintptr_t)d_in % 16 || (uintptr_t)d_out % 16) throw std::invalid_argument("label apply: the volumes must be 16-byte aligned");
    if (d_out != d_in) {
      const char *a = (const char*)d_in, *b = (const char*)d_out;
      const int64_t out_bytes = out_dtype == CFB_DTYPE_U64 ? 8 : in_bytes;
      if (a < b + voxels * out_bytes && b < a + voxels * in_bytes) throw std::invalid_argument("label apply: input and output overlap");
    }
    cudaStream_t s = (cudaStream_t)stream;
    const LtTable t = lt_table(d_workspace, table_slots);
    unsigned long long h[kLtStatWords];
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (h[kLtOverflow] || !h[kLtPlanned]) throw std::invalid_argument("label apply: the table in the workspace is incomplete or has no plan");
    if (h[kLtRenumbered] && out_dtype != CFB_DTYPE_U64) throw std::invalid_argument("label apply: renumbered labels need a uint64 output");
    if (in_dtype == CFB_DTYPE_U8) lt_launch_apply((const uint8_t*)d_in, voxels, t, d_out, out_dtype, s);
    else if (in_dtype == CFB_DTYPE_U32) lt_launch_apply((const uint32_t*)d_in, voxels, t, d_out, out_dtype, s);
    else lt_launch_apply((const uint64_t*)d_in, voxels, t, d_out, out_dtype, s);
    CFB_CUDA(cudaMemcpyAsync(h, t.stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    if (h[kLtMissing]) throw std::invalid_argument("label apply: the volume holds a label the table does not (another volume's table?)");
    return CFB_OK;
  });
}
