/*
 * chunkflow_b200 -- C-ABI of the H100-native `inference` hot path.
 *
 * Drop-in boundary for chunkflow's overlap-tile convnet inference.  The reference is
 * pure Python; each entry point names the reference interface it replaces
 * (paths relative to the reference tree, v1.1.7):
 *
 *   cfb_create / cfb_destroy      Inferencer.__init__ / __exit__
 *                                 chunkflow/flow/divid_conquer/inferencer.py:36-171,177-181
 *   cfb_set_weight / cfb_commit_weights
 *                                 PyTorch.__init__ weight loading
 *                                 chunkflow/flow/divid_conquer/patch/pytorch.py:48-63
 *   cfb_patch_mask                PatchMask / make_patch_mask
 *                                 chunkflow/flow/divid_conquer/patch/patch_mask.py:6-48
 *   cfb_patch_grid                Inferencer._construct_patch_slices_list   inferencer.py:255-292
 *   cfb_output_shape              Inferencer._update_parameters_for_input_chunk   inferencer.py:183-204
 *   cfb_infer_chunk_device/_host  Inferencer.__call__   inferencer.py:360-479
 *                                 (Chunk.cutout chunk/base.py:761-781, Chunk.blend chunk/base.py:792-807,
 *                                  PyTorch.__call__ patch/pytorch.py:98-119)
 *   cfb_patch_forward_host        PatchInferencer.__call__ plugin level
 *                                 patch/pytorch.py:98-119, patch/universal.py:60-69, patch/identity.py:30-51
 *   cfb_device_name               Inferencer.compute_device   inferencer.py:173-175
 *   cfb_watershed_device, cfb_region_graph_*, cfb_agglomerate_edges_host, cfb_relabel_device
 *                                 plugins/agglomerate.py:8-48 (execute -> waterz.agglomerate)
 *   cfb_contingency_*, cfb_evaluate_workspace
 *                                 Segmentation.evaluate   chunk/segmentation.py:33-67 (-> lib/gala/evaluate.py)
 *   cfb_label_table_*, cfb_label_apply_device
 *                                 Segmentation.remap / mask_fragments / mask_except   chunk/segmentation.py:69-109
 *   cfb_downsample_*              the `downsample` command   flow/flow.py:1545-1573 (-> lib/igneous/downsample.py)
 *   cfb_gaussian_filter_*         Chunk.gaussian_filter_2d   chunk/base.py:846-853 (`gaussian-filter`, flow/flow.py:1615-1630),
 *                                 plugins/gaussian_filter.py:7-23 (-> scipy.ndimage.gaussian_filter)
 *   cfb_median_filter_device      plugins/median_filter.py:4-7 (-> scipy.ndimage.median_filter)
 *   cfb_clahe_*                   plugins/clahe.py (-> cv2.createCLAHE(clipLimit, tileGridSize).apply)
 *
 * Plain pointers and sizes only -- no torch types.  Device pointers are raw CUDA device
 * addresses (e.g. torch.Tensor.data_ptr()) owned by the caller.  All functions return
 * CFB_OK (0) or a negative error code; cfb_last_error() returns the message of the last
 * failure on the calling thread.  There is NO CPU fallback: without a CUDA device every
 * compute entry point fails with CFB_ERR_CUDA.
 */
#ifndef CHUNKFLOW_B200_H_
#define CHUNKFLOW_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CFB_OK 0
#define CFB_ERR_INVALID_ARGUMENT (-1)
#define CFB_ERR_CUDA (-2)
#define CFB_ERR_WEIGHTS (-3)
#define CFB_ERR_OUTPUT_RANGE (-4) /* some output >= 1.0001 (reference inferencer.py:465-466) */
#define CFB_ERR_UNSUPPORTED (-5)
#define CFB_ERR_CAPACITY (-6) /* a caller-sized table is too small: call again with a larger one */

/* framework: which patch backend runs on the device */
#define CFB_FRAMEWORK_UNET3L 0   /* plain 3D U-Net of depth 2-4 (chunkflow_b200/convnet/unet3l.py), depth from the weights */
#define CFB_FRAMEWORK_IDENTITY 1 /* reference patch/identity.py: output = input patch */

/* precision of the convolution stack */
#define CFB_PRECISION_F32_SIMT 0   /* fp32 FFMA direct convolution (exact-order-free fp32) */
#define CFB_PRECISION_F16X3_UMMA 1 /* wgmma fp16 hi/lo split, fp32 accumulate (~fp32 accuracy) */
#define CFB_PRECISION_F16_UMMA 2   /* wgmma single-pass fp16, fp32 accumulate (reference --dtype float16) */
#define CFB_PRECISION_F16F8_UMMA 3 /* wgmma fp16 main product + ONE e4m3 (K = 32) product carrying both correction terms,
                                      fp32 accumulate: two tensor-core products per multiply instead of f16x3's three
                                      (csrc/act_format.cuh) */

/* test-time augmentation (`--augment`, reference inferencer.py:422-431 + transform.py).
 * REFERENCE reproduces the reference's arithmetic literally: its FlipLR / FlipUD call np.fliplr / np.flipud on
 * arr[..., z, :, :] of the 5-D (B, C, z, y, x) buffers, i.e. they reverse the CHANNEL and BATCH axes
 * (transform.py:30-52), so the average over its 8 sequences is
 *   1/4 * (n(x) + rev_c n(x) + T n(T x) + rev_c T n(T x)),   T = transpose y<->x, rev_c = output channels reversed.
 * SPATIAL is the evidently intended augmentation: the 8 combinations of {transpose} x {flip x} x {flip y}, each
 * undone on the output, averaged (an explicit opt-in; it does NOT reproduce the reference's numbers). */
#define CFB_AUGMENT_NONE 0
#define CFB_AUGMENT_REFERENCE 1
#define CFB_AUGMENT_SPATIAL 2

/* dtype of the input chunk */
#define CFB_DTYPE_U8 0
#define CFB_DTYPE_F32 1
#define CFB_DTYPE_U32 2 /* connected components on an integer segmentation */
#define CFB_DTYPE_U64 3 /* segmentation evaluation and clean-up: 64-bit label ids */
#define CFB_DTYPE_BOOL 4 /* downsample: a boolean segmentation (one byte per voxel), always strided */

typedef struct cfb_engine* cfb_handle;

typedef struct cfb_params {
  int32_t struct_size;             /* = sizeof(cfb_params), for ABI checks */
  int32_t device;                  /* CUDA device ordinal */
  int32_t framework;               /* CFB_FRAMEWORK_* */
  int32_t precision;               /* CFB_PRECISION_* */
  int32_t input_patch_size[3];     /* z, y, x */
  int32_t output_patch_size[3];    /* z, y, x (<= input; crop margin = (in-out)/2) */
  int32_t output_patch_overlap[3]; /* z, y, x */
  int32_t output_crop_margin[3];   /* z, y, x: margin of the output chunk that is dropped */
  int32_t num_input_channels;      /* must be 1 */
  int32_t num_output_channels;     /* channels returned (network may produce more; first N kept) */
  int32_t batch_size;              /* patches in flight per launch (scheduling hint) */
  int32_t mask_output_chunk;       /* 1: normalise by the accumulated weight volume */
  int32_t augment;                 /* CFB_AUGMENT_*: test-time augmentation (reference transform.py:114-156) */
  int32_t has_myelin_threshold;    /* 1: drop last channel, zero where it is >= threshold */
  float mask_myelin_threshold;
  int32_t check_output_range;      /* 1: fail with CFB_ERR_OUTPUT_RANGE like the reference assert */
} cfb_params;

const char* cfb_last_error(void);
int cfb_version(void);
/* Number of CUDA devices visible (0 if none / no driver). Never fails. */
int cfb_device_count(void);

/* Free / total bytes of device memory (used to size the number of patches in flight). */
int cfb_device_memory(int32_t device, int64_t* free_bytes, int64_t* total_bytes);

int cfb_create(const cfb_params* params, cfb_handle* out);
int cfb_destroy(cfb_handle h);
/* Name of the CUDA device the engine runs on (valid until cfb_destroy). */
const char* cfb_device_name(cfb_handle h);

/* Weights: fp32 host arrays in PyTorch state_dict layout, keyed by state_dict name
 * ("enc0.0.weight", "enc0.0.bias", ... "head.bias"). commit packs them for the kernels. */
int cfb_set_weight(cfb_handle h, const char* name, const float* host_data, int64_t numel);
int cfb_commit_weights(cfb_handle h);

/* Device-free: fp32 patch mask for (patch z,y,x ; overlap z,y,x) into host memory
 * (prod(patch) floats).  Replaces make_patch_mask, patch/patch_mask.py:15-48. */
int cfb_make_patch_mask(const int32_t patch_size[3], const int32_t overlap[3], float* host_out);

/* Copies the fp32 patch mask (prod(output_patch_size) floats) to host memory. */
int cfb_patch_mask(cfb_handle h, float* host_out);

/* Every call that takes a chunk shape (cz, cy, cx) returns CFB_ERR_INVALID_ARGUMENT for a chunk smaller than the
 * input patch, a dimension above INT32_MAX, or an output crop margin that leaves no output voxel. */

/* Patch grid for a chunk of the given size: writes the number of patches and, if
 * starts_zyx != NULL, up to `capacity` chunk-local input start triples (z,y,x per patch,
 * z-major then y then x, last patch per axis clamped). */
int cfb_patch_grid(cfb_handle h, int64_t cz, int64_t cy, int64_t cx,
                   int64_t* num_patches, int32_t* starts_zyx, int64_t capacity);

/* Output chunk shape (C, z, y, x) for an input chunk (z, y, x). */
int cfb_output_shape(cfb_handle h, int64_t cz, int64_t cy, int64_t cx, int64_t out_czyx[4]);

/* Whole-chunk inference, input and output resident in device memory.
 * d_in : (cz,cy,cx) uint8 or float32, contiguous; d_out: (C,oz,oy,ox) float32.
 * `stream` is a cudaStream_t (NULL = default stream).  Asynchronous unless
 * check_output_range is set (the range check synchronises the stream). */
int cfb_infer_chunk_device(cfb_handle h, const void* d_in, int32_t in_dtype,
                           int64_t cz, int64_t cy, int64_t cx, float* d_out, void* stream);

/* Same, host buffers: H2D copy of the chunk, inference, D2H copy of the result. */
int cfb_infer_chunk_host(cfb_handle h, const void* h_in, int32_t in_dtype,
                         int64_t cz, int64_t cy, int64_t cx, float* h_out);

/* One oversized chunk split across GPUs (BASELINE config #5; the reference has no counterpart, its unit of
 * parallelism is one process per GPU on independent chunks, distributed/kubernetes/deploy.yml:37):
 *   cfb_infer_slab_device     processes only the patches whose z-row index is in [zrow_begin, zrow_end) and leaves
 *                             d_out as the UN-normalised partial sum; d_weight (oz,oy,ox), if not NULL, receives this
 *                             slab's partial weight sum.
 *   cfb_slab_nonzero          the any-nonzero flag of the input of the last slab / chunk call (all ranks OR it to
 *                             reproduce the reference's all-zero shortcut, inferencer.py:387-393); synchronises.
 *   cfb_halo_add_device       d_dst[i] += d_src[i]: the owner of a plane adds the partial sums received from the
 *                             other ranks whose slabs overlap it (NCCL send/recv of the planes, then this kernel).
 *   cfb_weight_volume_device  planes [z_begin, z_end) of the weight volume (sum of the bump masks of ALL patches of
 *                             a (cz,cy,cx) chunk, reference inferencer.py:294-333; 1/W if `invert`): pure geometry,
 *                             so the owner computes it locally -- no weight halo is exchanged.
 *   cfb_normalize_device      d_out *= 1/d_weight (or *= d_weight if weight_is_inverse; NULL = no weight), the
 *                             reference's `< 1.0001` assertion (CFB_ERR_OUTPUT_RANGE, when check_output_range is set),
 *                             myelin masking; all_zero_input != 0 forces the result to zero. */
int cfb_infer_slab_device(cfb_handle h, const void* d_in, int32_t in_dtype,
                          int64_t cz, int64_t cy, int64_t cx,
                          int64_t zrow_begin, int64_t zrow_end,
                          float* d_out, float* d_weight, void* stream);
int cfb_slab_nonzero(cfb_handle h, int32_t* nonzero, void* stream);
int cfb_halo_add_device(float* d_dst, const float* d_src, int64_t count, void* stream);
int cfb_weight_volume_device(cfb_handle h, int64_t cz, int64_t cy, int64_t cx, int64_t z_begin, int64_t z_end,
                             int32_t invert, float* d_weight, void* stream);
int cfb_normalize_device(cfb_handle h, float* d_out, const float* d_weight, int32_t weight_is_inverse,
                         int64_t channels, int64_t oz, int64_t oy, int64_t ox, int32_t all_zero_input, void* stream);

/* PatchInferencer plugin level: `batch` input patches (batch,1,pz,py,px) float32 in
 * [0,1] on the host -> (batch,C,oz,oy,ox) float32 on the host, already cropped and
 * multiplied by the patch mask (reference patch/pytorch.py:112-113). */
int cfb_patch_forward_host(cfb_handle h, const float* h_patches, int32_t batch, float* h_out);

/* Plugin level for user-supplied patch backends (`-f universal`, framework='prebuilt';
 * reference patch/universal.py:43-69, inferencer.py:209-211,404-455).  The user's callable
 * maps host patches to host outputs that are ALREADY cropped and bump-masked; extract,
 * blend and normalise still run on the device:
 *   begin   : upload the chunk, build the patch grid, zero the accumulators
 *   extract : patches [first, first+nb) -> (nb,1,pz,py,px) float32 on the host
 *   blend   : (nb,C,oz,oy,ox) float32 masked outputs from the host -> accumulate
 *   end     : normalise (+ range check, myelin) and copy (C,oz,oy,ox) to the host */
int cfb_plugin_begin(cfb_handle h, const void* h_in, int32_t in_dtype, int64_t cz, int64_t cy, int64_t cx);
int cfb_plugin_extract(cfb_handle h, int64_t first, int32_t nb, float* h_patches);
int cfb_plugin_blend(cfb_handle h, int64_t first, int32_t nb, const float* h_masked_outputs);
int cfb_plugin_end(cfb_handle h, float* h_out);

/* Timing of the last cfb_infer_chunk_* call, CUDA events on the work stream (ms):
 * [0] total device time, [1] convnet kernels, [2] blend+normalise, [3] h2d, [4] d2h.
 * Kernel launches of the last call are returned through *launches. */
int cfb_last_timing(cfb_handle h, float ms[5], int64_t* launches);

/* Per-layer profiling (tracing aid; reference keeps only wall-clock per operator,
 * flow/flow.py:1926-1932).  When enabled every network kernel launch of the following
 * inference calls is bracketed by CUDA events on the work stream.  cfb_layer_timing
 * synchronises and reports, for up to `capacity` kernel classes: a name (<=31 chars),
 * total milliseconds and launch count accumulated since profiling was enabled. */
int cfb_set_profiling(cfb_handle h, int32_t enabled);
int cfb_layer_timing(cfb_handle h, int32_t capacity, int32_t* count, char (*names)[32], float* ms,
                     int64_t* launches);

/* Test hook: raw network output (before crop/mask) of one host patch, (Cnet,pz,py,px). */
int cfb_debug_net_forward_host(cfb_handle h, const float* h_patch, float* h_out);
/* Test hook: one step of the U-Net layer table run through the kernels of the engine's precision mode, on fp32 planar
 * host arrays.  The tensor-core modes convert the sources to the mode's activation format (a 128-channel tensor half-major)
 * and the results back; the cross-check switches CFB_NO_POOL_FUSION, CFB_SIMT_CONVT and CFB_NO_FUSED_TAIL are honoured as
 * in inference.  Shapes (nb patches, c = ca + cb channels, size = z, y, x of the step's input):
 *   CONV3            a (nb,ca,size) and b (nb,cb,size), two separate allocations concatenated as torch.cat([a, b]);
 *                    weight (cout,c,3,3,3), bias (cout) -> out (nb,cout,size); relu optional
 *   CONV3_POOL       the same, and pooled (nb,cout,z,y/2,x/2) = its (1,2,2) max pool
 *   CONVT            a (nb,ca,size), weight (ca,cout,1,2,2), bias (cout) -> out (nb,cout,z,2y,2x)
 *   MAXPOOL          a (nb,ca,size) -> out (nb,ca,z,y/2,x/2)
 *   FIRST            weight (16,1,3,3,3), bias (16) -> out (nb,16,size), ReLU; from a (nb,1,size), or, if chunk is
 *                    not NULL, from the uint8 (normalised by 1/255) or float32 chunk at in_origins
 *   HEAD_SIGMOID     a (nb,16,size), head_weight (head_channels,16), head_bias -> out (nb,head_channels,size)
 *   HEAD_BLEND       the same head, then crop, x mask (out_patch) x scale, accumulated into out (head_channels,out_size)
 *                    at out_origins (a patch may stick out of out_size: clipped)
 *   CONV3_HEAD_BLEND the 16 -> 16 CONV3 (ReLU) and HEAD_BLEND in one step: the fused epilogue on the tensor cores
 *   ROUND_TRIP       a (nb,ca,size) -> the mode's activation format -> out (nb,ca,size) */
#define CFB_LAYER_CONV3 0
#define CFB_LAYER_CONV3_POOL 1
#define CFB_LAYER_CONVT 2
#define CFB_LAYER_MAXPOOL 3
#define CFB_LAYER_FIRST 4
#define CFB_LAYER_HEAD_SIGMOID 5
#define CFB_LAYER_HEAD_BLEND 6
#define CFB_LAYER_CONV3_HEAD_BLEND 7
#define CFB_LAYER_ROUND_TRIP 8
typedef struct cfb_layer_args {
  int32_t struct_size; /* = sizeof(cfb_layer_args) */
  int32_t op;          /* CFB_LAYER_* */
  int32_t nb;
  int32_t size[3];
  int32_t ca, cb, cout, relu;
  const float* a;
  const float* b;
  const float* weight;
  const float* bias;
  const float* head_weight;
  const float* head_bias;
  int32_t head_channels;
  int32_t chunk_dtype; /* CFB_DTYPE_U8 or CFB_DTYPE_F32 */
  const void* chunk;
  int32_t chunk_size[3];
  int32_t out_patch[3], crop[3], out_size[3];
  const int32_t* in_origins;  /* (nb, 3) */
  const int32_t* out_origins; /* (nb, 3) */
  const float* mask;
  float scale;
  float* out;
  float* pooled;
} cfb_layer_args;
int cfb_debug_layer_host(cfb_handle h, const cfb_layer_args* args);

/* ---------------------------------------------------------------------------------------------
 * Operators either side of `inference`, on device memory (SURVEY.md section 8 f3): the chunk can stay in HBM
 * between operators.  Stand-alone entry points (no handle); every pointer is a device pointer on the current
 * device; work is enqueued on `stream` (a cudaStream_t, may be NULL).  Results are bit-identical to the reference's
 * numpy code.  Python mirror: chunkflow_b200/chunk/device.py (DeviceChunk).
 * ------------------------------------------------------------------------------------------- */
#define CFB_QUANTIZE_XY 0
#define CFB_QUANTIZE_Z 1

/* In-place Image.normalize_contrast (reference chunk/image/base.py:30-132) of a (z,y,x) uint8 image: per-section
 * 256-bin histogram (bin 0 ignored, 255 bins unless the value 255 occurs) -> clamping values at the clip fractions ->
 * float32 lookup table clipped to [minval,maxval], rounded half to even -> applied; then, as in the reference (the
 * whole-array branch is the `else` of its `for` loop), once more with the histogram of the WHOLE normalised array.
 * per_section == 0 does nothing, exactly like the reference.  0 <= minval <= maxval <= 255. */
int cfb_normalize_contrast_device(void* d_image, int64_t z, int64_t y, int64_t x, double lower_clip_fraction,
                                  double upper_clip_fraction, int32_t minval, int32_t maxval, int32_t per_section,
                                  void* stream);

/* In-place Chunk.maskout (reference chunk/base.py:811-829): chunk[c,z,y,x] *= mask[z/fz, y/fy, x/fx], the mask being
 * (z/fz, y/fy, x/fx) voxels at an integer multiple (fz,fy,fx) of the chunk's voxel size.  dtype pairs as numpy allows
 * them in place: (U8 chunk, U8/bool mask), (F32 chunk, U8/bool mask), (F32 chunk, F32 mask). */
int cfb_maskout_device(void* d_chunk, int32_t chunk_dtype, int64_t channels, int64_t z, int64_t y, int64_t x,
                       const void* d_mask, int32_t mask_dtype, int64_t fz, int64_t fy, int64_t fx, void* stream);

/* Chunk.crop_margin (reference chunk/base.py:691-726): d_dst (channels, z-m0-m3, y-m1-m4, x-m2-m5) receives
 * src[..., m0:z-m3, m1:y-m4, m2:x-m5]; margin = {-z,-y,-x,+z,+y,+x} (the 3-element form is m3..5 = m0..2). */
int cfb_crop_margin_device(const void* d_src, int32_t dtype, int64_t channels, int64_t z, int64_t y, int64_t x,
                           const int64_t margin[6], void* d_dst, void* stream);

/* AffinityMap.quantize (reference chunk/affinity_map/base.py:33-57): (channels,z,y,x) float32 -> (z,y,x) uint8,
 * CFB_QUANTIZE_XY: uint8(((a[0] + a[1]) / 2) * 255), CFB_QUANTIZE_Z: uint8(a[channels-1] * 255); float32
 * arithmetic, C truncation. */
int cfb_quantize_device(const float* d_affinity, int64_t channels, int64_t z, int64_t y, int64_t x, int32_t mode,
                        uint8_t* d_out, void* stream);

/* `connected-components` (SURVEY.md section 8 f4): Chunk.connected_component (reference chunk/base.py:128-137) =
 * [Chunk.threshold: array > threshold (:728-737)] + cc3d.connected_components(seg, connectivity).  d_in: (z,y,x) uint8 / uint32
 * labels (0 = background; equal non-zero values connect) or float32 (thresholded first); connectivity 6 / 18 / 26;
 * d_labels: (z,y,x) uint32, components numbered 1..N in the order of their first voxel in a raster scan (x fastest), like cc3d.
 * d_workspace: cfb_connected_components_workspace(z,y,x) bytes of device memory.  num_labels (host, may be NULL; when given the
 * stream is synchronised) receives N. */
int cfb_connected_components_device(const void* d_in, int32_t in_dtype, int64_t z, int64_t y, int64_t x, float threshold,
                                    int32_t connectivity, uint32_t* d_labels, void* d_workspace, uint32_t* num_labels,
                                    void* stream);
int64_t cfb_connected_components_workspace(int64_t z, int64_t y, int64_t x);

/* `agglomerate` (SURVEY.md section 8 f4): the reference's plugin (chunkflow/plugins/agglomerate.py:8-48) hands the affinity
 * map to waterz.agglomerate(affs, [threshold], fragments=, aff_threshold_low=, aff_threshold_high=,
 * scoring_function='OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>') -- watershed fragments, region graph,
 * hierarchical merging.  waterz is a third-party package that is not vendored in the reference tree; its published algorithm
 * is restated in oracle/agglomeration_oracle.py ("parity unpinned").  Four steps, the voxel passes on the device:
 *
 * d_affs: (3, z, y, x) float32.  flip_channel != 0: the channels are in chunkflow's order x, y, z (the plugin's
 * `flip_channel`, agglomerate.py:26-29: waterz wants z, y, x) and are read in reverse instead of being copied.
 *
 * cfb_watershed_device: steepest-ascent watershed (waterz backend/watershed.hpp; Zlateski & Seung, arXiv:1505.00249) ->
 * d_fragments (z,y,x) uint32, basins numbered 1..N in raster order of their first voxel, 0 = voxels whose strongest edge does
 * not exceed aff_threshold_low.  Plateau interiors drain towards the neighbour one breadth-first step closer to a plateau
 * corner (order independent; the sequential code's queue order is not reproduced, see the oracle).  d_workspace:
 * cfb_watershed_workspace(z,y,x) bytes.  num_fragments (host, may be NULL; the stream is synchronised either way). */
int64_t cfb_watershed_workspace(int64_t z, int64_t y, int64_t x);
int cfb_watershed_device(const float* d_affs, int32_t flip_channel, int64_t z, int64_t y, int64_t x, float aff_threshold_low,
                         float aff_threshold_high, uint32_t* d_fragments, void* d_workspace, uint32_t* num_fragments,
                         void* stream);

/* Region graph (waterz backend/region_graph.hpp with the MeanAffinity statistics): for every pair of touching fragments
 * (6-neighbourhood, ids != 0) the SUM of the affinities on the faces between them, in 2^-30 fixed point (each affinity clamped
 * to [0,1], NaN = 0, rounded to nearest even: the sum does not depend on the order of the atomics), and their COUNT.  Built in
 * an open-addressing table of `table_slots` (a power of two) slots inside d_workspace (cfb_region_graph_workspace(table_slots)
 * bytes); returns CFB_ERR_CAPACITY when the table is too full -- call again with more slots.  *num_edges = pairs found.
 * cfb_region_graph_read copies the edges to the host, sorted by (u, v), u < v. */
int64_t cfb_region_graph_workspace(int64_t table_slots);
int cfb_region_graph_device(const float* d_affs, int32_t flip_channel, const uint32_t* d_fragments, int64_t z, int64_t y, int64_t x,
                            void* d_workspace, int64_t table_slots, int64_t* num_edges, void* stream);
int cfb_region_graph_read(void* d_workspace, int64_t table_slots, int64_t num_edges, uint32_t* h_u, uint32_t* h_v,
                          uint64_t* h_sum_fixed, uint32_t* h_count, void* stream);

/* The merge loop (waterz backend/IterativeRegionMerging.hpp, scoring function OneMinus<MeanAffinity>), on the HOST like
 * waterz's own: repeatedly merge the edge with the smallest score 1 - sum / (count * 2^30) (ties: the edge holding the smallest
 * original (u, v) pair first) until the smallest score reaches `threshold`; a merged cluster is known by its smallest id,
 * edges to a common neighbour pool their statistics.  root_of[i], i < num_nodes (= largest fragment id + 1), receives the id node i ends up with
 * (root_of[0] == 0).  No GPU involved. */
int cfb_agglomerate_edges_host(int64_t num_nodes, int64_t num_edges, const uint32_t* u, const uint32_t* v,
                               const uint64_t* sum_fixed, const uint32_t* count, float threshold, uint32_t* root_of);

/* Histogram region graph (waterz's HistogramQuantileAffinity statistics): for every pair of touching fragments (the faces
 * and channels of cfb_region_graph_device) the number of faces whose affinity a -- clamped to [0,1], NaN = 0, float32 --
 * falls in bin min((int)(a * bins), bins - 1), 2 <= bins <= 256, and the largest clamped affinity.  Two passes over the
 * faces: the pair table, then a table of (pair, bin) counts of 2 x table_slots slots, both inside d_workspace
 * (cfb_region_graph_hist_workspace(table_slots) bytes); CFB_ERR_CAPACITY when either is too full -- call again with more slots.
 * *num_edges = pairs, *num_entries = non-empty (pair, bin) counts.  cfb_region_graph_hist_read copies them to the host:
 * edges sorted by (u, v), u < v, with their maxima; h_offsets (num_edges + 1) delimits each edge's run of h_bins / h_counts,
 * sorted by bin. */
int64_t cfb_region_graph_hist_workspace(int64_t table_slots);
int cfb_region_graph_hist_device(const float* d_affs, int32_t flip_channel, const uint32_t* d_fragments, int64_t z, int64_t y,
                                 int64_t x, int32_t bins, void* d_workspace, int64_t table_slots, int64_t* num_edges,
                                 int64_t* num_entries, void* stream);
int cfb_region_graph_hist_read(void* d_workspace, int64_t table_slots, int64_t num_edges, int64_t num_entries, uint32_t* h_u,
                               uint32_t* h_v, uint64_t* h_offsets, uint8_t* h_bins, uint32_t* h_counts, float* h_max, void* stream);

/* The merge loop with OneMinus<HistogramQuantileAffinity<RegionGraphType, quantile, ScoreValue, num_bins, init_with_max>>,
 * on the host.  Edge i holds the bins offsets[i] .. offsets[i+1] (strictly increasing, < num_bins, non-zero counts) and, when
 * init_with_max, maxima[i] in [0, 1] (maxima may be NULL otherwise).  score = 1 - (q + 0.5) / num_bins, q the first bin whose
 * cumulative count reaches min(floor(quantile * n / 100) + 1, n) of the n faces; with init_with_max, an edge that has never
 * been pooled scores 1 - its maximum.  Pooled edges add their histograms and keep the anchor of the one that comes first in
 * (score, anchor) order.  Otherwise as cfb_agglomerate_edges_host (rules: oracle/agglomeration_oracle.py). */
int cfb_agglomerate_quantile_host(int64_t num_nodes, int64_t num_edges, const uint32_t* u, const uint32_t* v, const uint64_t* offsets,
                                  const uint8_t* bins, const uint32_t* counts, const float* maxima, int32_t quantile,
                                  int32_t num_bins, int32_t init_with_max, float threshold, uint32_t* root_of);

/* d_out[i] = d_map[d_labels[i]] (labels >= map_size pass through): applies root_of to the fragments. */
int cfb_relabel_device(const uint32_t* d_labels, int64_t n, const uint32_t* d_map, int64_t map_size, uint32_t* d_out,
                       void* stream);

/* `evaluate-segmentation` (DESIGN.md section 0, row f5): Segmentation.evaluate(groundtruth, size_threshold) (reference
 * chunk/segmentation.py:33-67, called by flow/flow.py:1519-1542) scores a segmentation against ground truth with the vendored
 * gala metrics (reference lib/gala/evaluate.py).  With c_ij the number of voxels labelled i in the segmentation and j in the
 * ground truth (the contingency table, contingency_table :212-249):
 *   rand / adjusted rand / Fowlkes-Mallows index  rand_values (:1183-1223) and :1248, :1274-1275, :1300, 0 an ordinary label:
 *       a = (S1 - n) / 2, b = (S2 - S1) / 2, c = (S3 - S1) / 2, d = (S1 + n^2 - S2 - S3) / 2 with S1 = sum c^2, S2 = sum of the
 *       squared row sums, S3 = sum of the squared column sums;
 *   variation of information  vi -> split_vi -> vi_tables (:623-691, :1049-1101), voxels with a 0 on either side ignored:
 *       ((xl(r') - xl(c)) + (xl(s') - xl(c))) / N', xl(v) = sum v log2 v over those voxels' table, rows r', columns s';
 *   edit distance  raw_edit_distance (:183-209): (K - N_seg, 0.0), K = pairs with both ids != 0 and c > size_threshold,
 *       N_seg = distinct non-zero segmentation ids.  The second element is always 0 in the reference (it slices the rows of a
 *       1 x N matrix); kept.
 * 0/0 gives NaN, as in the reference.  Ids are compared as the uint64 values numpy's astype(np.uint64) gives; every uint64 is
 * a legal id (the reference itself fails on ids of about 2^40 and more; here they are scored like any other).
 *
 * cfb_contingency_device  d_seg, d_gt: (z,y,x) volumes of CFB_DTYPE_U8 / U32 / U64 ids (n < 2^32 voxels).  Builds the table
 *                         of (seg id, gt id) -> count in d_workspace (cfb_evaluate_workspace(table_slots) bytes, table_slots
 *                         a power of two below 2^31) and the statistics of all thresholds; *num_pairs = entries.  Returns
 *                         CFB_ERR_CAPACITY when the table is too full -- call again with more slots.  Synchronises.
 * cfb_contingency_scores  statistics + scores of the table in d_workspace for one size_threshold (compared like the
 *                         reference's `r.data <= size_threshold`); a threshold sweep reuses the table.  Synchronises.
 * cfb_contingency_read    the table as (seg id, gt id, count) triples sorted by (seg, gt) into host arrays of num_pairs. */
typedef struct cfb_seg_scores {
  int32_t struct_size;            /* = sizeof(cfb_seg_scores), for ABI checks */
  int32_t reserved;
  uint64_t n;                     /* voxels */
  uint64_t sum_sq_pairs;          /* S1 */
  uint64_t sum_sq_rows;           /* S2 */
  uint64_t sum_sq_cols;           /* S3 */
  uint64_t n_both_nonzero;        /* N': voxels with both ids != 0 */
  uint64_t seg_ids;               /* N_seg: distinct non-zero segmentation ids */
  uint64_t gt_ids;                /* N_gt: distinct non-zero ground-truth ids */
  uint64_t pairs;                 /* entries of the contingency table */
  uint64_t pairs_over_threshold;  /* K(size_threshold) */
  double size_threshold;
  double xlog_pairs;              /* xl(c) over the pairs with both ids != 0 */
  double xlog_rows;               /* xl(r') */
  double xlog_cols;               /* xl(s') */
  double rand_index, adjusted_rand_index, variation_of_information, fowlkes_mallows_index;
  double false_merges, false_splits;  /* edit distance */
} cfb_seg_scores;

int64_t cfb_evaluate_workspace(int64_t table_slots);
int cfb_contingency_device(const void* d_seg, int32_t seg_dtype, const void* d_gt, int32_t gt_dtype, int64_t z, int64_t y,
                           int64_t x, void* d_workspace, int64_t table_slots, int64_t* num_pairs, void* stream);
int cfb_contingency_scores(void* d_workspace, int64_t table_slots, double size_threshold, cfb_seg_scores* out, void* stream);
int cfb_contingency_read(void* d_workspace, int64_t table_slots, int64_t num_pairs, uint64_t* h_seg, uint64_t* h_gt,
                         uint32_t* h_count, void* stream);

/* Segmentation clean-up (DESIGN.md section 0, row f6): Segmentation.mask_fragments(t) / mask_except(ids) / remap(base_id)
 * (reference chunk/segmentation.py:69-109; the first two are the `mask-out-objects` command, flow/flow.py:2015-2050).  The
 * reference delegates to fastremap (unique, mask, mask_except, renumber), a third-party package outside the reference tree:
 * its behaviour is restated (oracle/relabel_oracle.py), the reference's own code around it is pinned by golden vectors.
 *   dust       every id whose voxel count is <= t becomes 0 (`<=`, as the reference's code has it, not its help text);
 *   keep-list  every id that is not listed becomes 0; listed ids that do not occur are ignored; an empty list masks all;
 *   renumber   the surviving non-zero ids become 1..N in the order of their first voxels in a C-order raster scan, plus
 *              base_id; 0 stays 0; the output is uint64.  Masking never reorders first voxels, so the three compose.
 * Every uint64 is a legal id.  Volumes hold at most 2^32 - 2 voxels (first-voxel indices are 32-bit) and are 16-byte aligned.
 *
 * cfb_label_table_workspace  bytes of d_workspace for a volume of `voxels` and a table of table_slots (a power of two in
 *                            [32, 2^31)).
 * cfb_label_table_device     one read of the (z,y,x) volume of CFB_DTYPE_U8 / U32 / U64 ids builds
 *                            id -> (voxel count, linear index of the first voxel) in d_workspace; *num_labels = entries (0
 *                            included when it occurs).  CFB_ERR_CAPACITY when the table is too full -- call again with more
 *                            slots.  Synchronises.
 * cfb_label_table_read       the table as host arrays of num_labels, ids ascending.
 * cfb_label_table_plan       writes every entry's new value for any combination of use_dust (count <= dust_threshold),
 *                            a keep-list of num_keep ids in device memory (num_keep < 0: none) and renumber (+ base_id;
 *                            base_id + N > 2^64 - 1 is refused).  *num_dust = entries failing the dust test (0 included: the
 *                            first number mask_fragments prints), *num_survivors = non-zero ids that stay non-zero, *new_max =
 *                            the maximum of the relabelled volume (0 when nothing survives, whatever base_id: the value the
 *                            reference returns).  No voxel is read.  Synchronises.
 * cfb_label_apply_device     second read of the volume, one write: d_out[i] = new value of d_in[i].  out_dtype is in_dtype
 *                            (d_out may then be d_in) or CFB_DTYPE_U64, which a renumbering plan requires.  Synchronises. */
int64_t cfb_label_table_workspace(int64_t voxels, int64_t table_slots);
int cfb_label_table_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, void* d_workspace,
                           int64_t table_slots, int64_t* num_labels, void* stream);
int cfb_label_table_read(void* d_workspace, int64_t table_slots, int64_t num_labels, uint64_t* h_ids, uint32_t* h_counts,
                         uint32_t* h_first, void* stream);
int cfb_label_table_plan(void* d_workspace, int64_t table_slots, int64_t voxels, int32_t use_dust, int64_t dust_threshold,
                         const uint64_t* d_keep_ids, int64_t num_keep, int32_t renumber, uint64_t base_id, int64_t* num_dust,
                         int64_t* num_survivors, uint64_t* new_max, void* stream);
int cfb_label_apply_device(const void* d_in, int32_t in_dtype, int64_t voxels, void* d_workspace, int64_t table_slots,
                           void* d_out, int32_t out_dtype, void* stream);

/* `downsample` (DESIGN.md section 0, row f7): the reference's command (flow/flow.py:1545-1573) averages a uint8 image and
 * mode-pools an integer or boolean segmentation by a factor (fz, fy, fx) of the (z,y,x) C-order volume.  It calls tinybrain,
 * a third-party package outside the reference tree (parity unpinned); the arithmetic pinned here, bit for bit, is the
 * reference's vendored numpy downsampler (lib/igneous/downsample.py), restated in oracle/downsample_oracle.py.  The output
 * of every level is ceil(extent / factor) per axis, except where a 2x2 step rounds an odd side up (below).
 *
 * cfb_downsample_average_device  downsample_with_averaging (:103-125): out = floor(block sum / voxels in the block), the
 *     blocks at the far edges clipped to the voxels that exist; that is the reference's float32 sum, float64 division and
 *     cast, for blocks of at most 65793 voxels (65793 * 255 < 2^24).  Larger blocks and factors below one return
 *     CFB_ERR_INVALID_ARGUMENT.  (1,1,1) copies the input.
 * cfb_downsample_segmentation_device  downsample_segmentation (:154-253), one level after the other from the element kind,
 *     the level's shape and the remaining factor f:
 *       all f == 1                                    done (no level: the input is copied);
 *       CFB_DTYPE_BOOL, or prod(f) not a power of two stride  out = in[::fz, ::fy, ::fx]  (:429-441), the last level;
 *       no f == 1, every extent even                  countless3d (:326-400), then f // 2;
 *       some f == 1                                   countless2d (:256-295) on the other two axes, the first axis with
 *                                                     f == 1 preserved, then f // 2 with the preserved axis kept at 1;
 *       otherwise (an odd extent)                     stride.
 *     countless2d: an odd side first gets a copy of its first row in front (odd_to_even2d :54-92), so output j reads inputs
 *     (max(2j - 1, 0), 2j); with a, b, c, d the pair's (lo,lo), (lo,hi), (hi,lo), (hi,hi) voxels: a if a == b or a == c, else
 *     b if b == c, else d.  countless3d, the 8 voxels in (z,y,x) ndindex order: the first value seen >= 4 times, else >= 3
 *     times, else >= 2 times among the first 7 voxels, else the 8th voxel.
 *     Kept quirks: the reference offsets ids by +1 in the stored width and takes 0 as "no pick", so the all-ones id
 *     (2^32 - 1, 2^64 - 1) never counts as a pick in countless3d, nor in countless2d for CFB_DTYPE_U64 (it widens 32-bit
 *     ids first).  A 2x2 step halves both other axes even when one of them has f == 1 -- its f // 2 is then 0, which the
 *     reference refuses, and so is the factor here.
 *     Deviations: the reference recurses with factor / 2, a float, and raises on every second level; here f // 2 is used,
 *     so that higher powers of two (4,4,4), (1,4,4), ... run level after level as its documentation intends.  The 2x2 step
 *     also takes the 3-D arrays on which the reference's raises.
 *     Refused with CFB_ERR_INVALID_ARGUMENT before any kernel: a factor below one, a product above 2^31 - 1, and every
 *     factor whose recursion reaches a factor of 0 ((1,1,2), (1,2,4), (2,2,4) on even shapes, ...).
 * cfb_downsample_workspace  the plan of a segmentation factor without a device: the output shape and the bytes of device
 *     memory the intermediate levels need (0 for one level); CFB_ERR_INVALID_ARGUMENT when the factor is refused.
 * dtype: CFB_DTYPE_U32 (also int32 volumes holding uint32 ids), CFB_DTYPE_U64 (also the bit pattern of int64 volumes) or
 * CFB_DTYPE_BOOL.  The input is only read; it may start at any address; input, output and workspace must not overlap. */
int cfb_downsample_average_device(const uint8_t* d_in, int64_t z, int64_t y, int64_t x, const int64_t factor[3], uint8_t* d_out,
                                  void* stream);
int cfb_downsample_workspace(int32_t dtype, int64_t z, int64_t y, int64_t x, const int64_t factor[3], int64_t out_zyx[3],
                             int64_t* workspace_bytes);
int cfb_downsample_segmentation_device(const void* d_in, int32_t dtype, int64_t z, int64_t y, int64_t x, const int64_t factor[3],
                                       void* d_workspace, void* d_out, void* stream);

/* `gaussian-filter` and the median filter (DESIGN.md section 0, row f8): the reference calls scipy.ndimage.gaussian_filter
 * (Chunk.gaussian_filter_2d, chunk/base.py:846-853; plugins/gaussian_filter.py:7-23) and scipy.ndimage.median_filter
 * (plugins/median_filter.py:4-7); the results here are bit-identical to scipy's on uint8 and float32, restated in
 * oracle/filters_oracle.py.  The chunk is (c, z, y, x) C-order, c = 1 for a 3-D chunk; dtype CFB_DTYPE_U8 or CFB_DTYPE_F32.
 *
 * cfb_gaussian_filter_device  in place: every z section is filtered on its own, one 1-D pass per axis in the order c, y, x;
 *     the channel pass mixes the channels of a section, as the reference does on a 4-D chunk.  w_<axis>[0..r_<axis>] are the
 *     float64 weights of scipy's kernel at truncate 4, w[0] the centre: radius r = int(4 sigma + 0.5),
 *     w = exp(-0.5 / sigma^2 * k^2) for k = -r..r, divided by their sum -- computed by the CALLER with numpy (numpy's and
 *     libm's exp may differ in the last bit).  A null w_<axis> with r_<axis> = 0 means no pass along that axis (scipy skips
 *     sigma <= 1e-15).  Per element, in float64, every operation rounded on its own: t = x[i] * w[0], then
 *     t = t + (x[i-j] + x[i+j]) * w[j] for j = r .. 1, indices reflected (d c b a | a b c d | d c b a, period 2n); then a cast
 *     to the chunk's type (uint8: toward zero, float32: to nearest) that the next pass reads.  r is 0 .. 64.
 *     d_workspace: cfb_gaussian_filter_workspace bytes (a batch of whole sections), not overlapping the chunk.
 * cfb_median_filter_device  out = element V / 2 of the sorted window of V = prod(size) elements (at most 125; each extent
 *     1 .. 125); the window of extent s spans offsets -(s / 2) .. s - 1 - (s / 2).  mode: CFB_FILTER_REFLECT (scipy 'reflect',
 *     'grid-mirror'), _NEAREST, _MIRROR (d c b | a b c d | c b a; one element mirrors onto itself), _WRAP ('wrap',
 *     'grid-wrap'), _CONSTANT (the value 0; 'constant', 'grid-constant').  size (1, 3, 1, 1) -- scipy's (3, 1, 1) on a 3-D
 *     chunk -- reads the chunk once.  Input and output must not overlap.  Outside the bit-identity claim: float32 NaN, and
 *     the sign of a zero in a tie of +0 and -0.
 * Sizes, radii and windows out of range return CFB_ERR_INVALID_ARGUMENT before any kernel runs.  64-bit indices; any address. */
#define CFB_FILTER_REFLECT 0
#define CFB_FILTER_NEAREST 1
#define CFB_FILTER_MIRROR 2
#define CFB_FILTER_WRAP 3
#define CFB_FILTER_CONSTANT 4
int cfb_gaussian_filter_workspace(int32_t dtype, int64_t c, int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes);
int cfb_gaussian_filter_device(void* d_data, int32_t dtype, int64_t c, int64_t z, int64_t y, int64_t x, const double* w_c,
                               int32_t r_c, const double* w_y, int32_t r_y, const double* w_x, int32_t r_x, void* d_workspace,
                               int64_t workspace_bytes, void* stream);
int cfb_median_filter_device(const void* d_in, int32_t dtype, int64_t c, int64_t z, int64_t y, int64_t x, const int64_t size[4],
                             int32_t mode, void* d_out, void* stream);

/* `clahe` (DESIGN.md section 0, row f9): the reference's plugins/clahe.py runs cv2.createCLAHE(clipLimit, tileGridSize).apply
 * on every z section of a uint8 image; the results here are bit-identical to OpenCV's, restated in oracle/clahe_oracle.py.
 * The chunk is uint8 (z, y, x) C-order; every section is equalized on its own.  tiles_x, tiles_y: cv2's tileGridSize, x first.
 *   padding   none when x % tiles_x == 0 and y % tiles_y == 0, else tiles_y - y % tiles_y rows at the bottom and
 *             tiles_x - x % tiles_x columns at the right (OpenCV pads both), BORDER_REFLECT_101 (d c b | a b c d | c b a),
 *             tiles of th x tw = T pixels of the padded section;
 *   clipping  clip_limit > 0: cl = max((int)(clip_limit * T / 256), 1) in double (out of the int32 range: INT32_MIN, as x86
 *             casts, so cl = 1); each tile's 256-bin histogram is clipped at cl, the clipped count spread over the bins
 *             (count / 256 to every bin, one more to bins 0, step, 2 step, ... while count % 256 lasts,
 *             step = max(256 / (count % 256), 1)).  clip_limit <= 0: no clipping;
 *   LUT       lut[v] = sat_u8(rint(float(cumsum(v)) * (255.f / T)));
 *   output    float32, every operation rounded on its own: txf = x * (1.f / tw) - 0.5f, tx1 = floor(txf), xa = txf - tx1,
 *             tx2 = min(tx1 + 1, tiles_x - 1), tx1 = max(tx1, 0), the same along y, and
 *             sat_u8(rint((L11 (1 - xa) + L12 xa) (1 - ya) + (L21 (1 - xa) + L22 xa) ya)), Lab = lut of tile (ty_a, tx_b).
 * cfb_clahe_workspace  bytes of d_workspace (the tile LUTs of a batch of sections; 0 for tiles of at most 64 pixels, whose
 *     LUT entries are computed where they are read).  No device needed.
 * cfb_clahe_device  d_out must not overlap d_in, nor the workspace either.  A section side above 2^24 pixels, a padded section
 *     above INT32_MAX pixels, or tiles_x / tiles_y below 1 return CFB_ERR_INVALID_ARGUMENT before any kernel runs.
 *     64-bit indices; any address. */
int cfb_clahe_workspace(int64_t z, int64_t y, int64_t x, int32_t tiles_x, int32_t tiles_y, int64_t* workspace_bytes);
int cfb_clahe_device(const void* d_in, void* d_out, int64_t z, int64_t y, int64_t x, double clip_limit, int32_t tiles_x,
                     int32_t tiles_y, void* d_workspace, int64_t workspace_bytes, void* stream);

/* `mesh` (reference flow/flow.py:2087-2135, flow/mesh.py -> zmesh): marching cubes of every object of a (z, y, x) segmentation,
 * restated in oracle/mesh_oracle.py (zmesh is not vendored: its meshes are not reproduced, parity unpinned).
 *   cubes     one per 2 x 2 x 2 group of voxel centres: z < Z-1, y < Y-1, x < X-1 (open, close = 0), or from -1 to Z-1 along
 *             every axis with everything outside the chunk 0 (close != 0: every object comes out watertight).  For every
 *             distinct id L among a cube's corners that is neither 0 nor among the d_skip_ids, the case is the mask of the
 *             corners equal to L (corner c at dz, dy, dx = c >> 2 & 1, c >> 1 & 1, c & 1); its triangles come from one
 *             256-case table built face by face (oracle/mesh_oracle.py), counter-clockwise seen from outside L.
 *   vertices  one per (object, cut edge): on the cut axis at (i + 1) * voxel size, on the others at (i + 0.5) * voxel size,
 *             for the edge's lower voxel i; float32, columns x, y, z.  Numbered in ascending order of the edge key
 *             ((z + 1) * (Y + 2) + (y + 1)) * (X + 2) + (x + 1)) * 3 + axis (0 x, 1 y, 2 z).  Faces in raster order of their
 *             cube, then in table order.
 * cfb_mesh_workspace  bytes of d_workspace (the counts) for a volume.  No device needed.
 * cfb_mesh_count_device  the (cube, object) pairs with a non-empty case, their triangles and the vertices (synchronises the
 *     stream).  dtype CFB_DTYPE_U32 or CFB_DTYPE_U64; d_skip_ids: num_skip ids on the device, ascending.  2^32 or more
 *     triangles or vertices return CFB_ERR_INVALID_ARGUMENT.
 * cfb_mesh_buffer_bytes  bytes of d_buffer for those counts.  No device needed.
 * cfb_mesh_device  after the count, with the same arguments, the workspace it filled and its counts: every mesh, welded on the
 *     device into d_buffer; *num_objects = the objects meshed.  voxel_size is (z, y, x).  Synchronises the stream.
 * cfb_mesh_read  the meshes to the host, objects in ascending order of id: object o has the faces face_offsets[o] ..
 *     face_offsets[o + 1] (rows of faces, indices into its own vertices) and the vertices vertex_offsets[o] ..
 *     vertex_offsets[o + 1] (rows of vertices).  object_ids holds num_objects entries, the offsets num_objects + 1, faces
 *     num_triangles rows and vertices num_vertices rows, the counts of cfb_mesh_count_device.
 * cfb_mesh_simplify_host  a restated Garland-Heckbert edge collapse of one mesh, fully ordered (rules:
 *     oracle/mesh_oracle.py simplify).  Face quadrics of the unit-normal planes, unweighted, in float64; the ends of an
 *     edge used by one face only (an open border) are locked.  Candidates: every edge not locked at both ends, placed at its
 *     locked end or at the first of (v_a, v_b, midpoint) with the least error, the error being the cost.  Collapsed in
 *     ascending (cost, a, b) order with lazy re-evaluation, a < b surviving with the summed quadric and re-queueing the edges
 *     of a and of its neighbours (so that a refused collapse is tried again once its surroundings change), unless that breaks the
 *     link condition, flips or degenerates a face that stays, or repeats a face's vertex set.  Stops at
 *     ceil(num_faces / simplification_factor) faces or when the cheapest cost exceeds max_simplification_error^2.  Faces
 *     keep their order, vertices are renumbered in order of first use; out_vertices and out_faces have room for the input.
 *     simplification_factor <= 1 copies the mesh unchanged.  No device needed. */
int cfb_mesh_workspace(int64_t z, int64_t y, int64_t x, int32_t close, int64_t* workspace_bytes);
int cfb_mesh_count_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const uint64_t* d_skip_ids,
                          int64_t num_skip, int32_t close, void* d_workspace, int64_t* num_pairs, int64_t* num_triangles,
                          int64_t* num_vertices, void* stream);
int cfb_mesh_buffer_bytes(int64_t num_pairs, int64_t num_triangles, int64_t num_vertices, int64_t* buffer_bytes);
int cfb_mesh_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const uint64_t* d_skip_ids, int64_t num_skip,
                    int32_t close, const double* voxel_size, void* d_workspace, int64_t num_pairs, int64_t num_triangles,
                    int64_t num_vertices, void* d_buffer, int64_t buffer_bytes, int64_t* num_objects, void* stream);
int cfb_mesh_read(void* d_buffer, int64_t num_pairs, int64_t num_triangles, int64_t num_vertices, int64_t num_objects, uint64_t* object_ids,
                  int64_t* face_offsets, int64_t* vertex_offsets, uint32_t* faces, float* vertices, void* stream);
int cfb_mesh_simplify_host(int64_t num_vertices, const float* vertices, int64_t num_faces, const uint32_t* faces,
                           int64_t simplification_factor, double max_simplification_error, int64_t* out_num_vertices,
                           float* out_vertices, int64_t* out_num_faces, uint32_t* out_faces);

/* `skeletonize` (reference plugins/skeletonize.py -> kimimaro.skeletonize): a TEASAR skeleton of every object of a (z, y, x)
 * segmentation, restated in oracle/skeleton_oracle.py (kimimaro is not vendored: its skeletons are not reproduced, parity
 * unpinned).  dtype CFB_DTYPE_U32 or CFB_DTYPE_U64; voxel_size is (z, y, x), positive; the chunk has fewer than 2^32 voxels.
 * Every error names the rule it broke in cfb_last_error.
 * cfb_skeleton_workspace  bytes of d_workspace for a volume (about 30 bytes per voxel).  No device needed.
 * cfb_edt_workspace  bytes of d_workspace for the distance transform alone (16 bytes per voxel).  No device needed.
 * cfb_edt_device  d_dbf (float32, n) = the distance of every voxel to the nearest voxel of another id, outside the chunk being
 *     0 (0 for id 0), in physical units.  d_workspace: cfb_edt_workspace bytes.
 * cfb_skeleton_count_device  the distance transform and the objects (26-connected components of one non-zero id that is not
 *     among the num_skip ascending d_skip_ids and has at least dust_threshold voxels) into d_workspace -> *num_objects, their
 *     *num_voxels and the *buffer_bytes of d_buffer for cfb_skeleton_device (synchronises the stream).
 * cfb_skeleton_device  after the count, with the same labels and workspace (one call per count: it overwrites the counts, and a
 *     second call is refused): params = (scale, const, pdrf_scale), every one finite and >= 0, pdrf_exponent 1..16, and
 *     (pdrf_scale + 1) * diagonal step * z * y * x * (1 + 2^-19) < 2^53 * the smallest voxel size, which keeps the geodesic
 *     field finite and strictly increasing along every step.  -> *num_skeleton_voxels; stats (8 doubles, may be null) =
 *     relaxation sweeps, rounds, paths, skeleton voxels, ms of the relaxation and parents, of the sort, of the rounds, and of the
 *     trace kernels alone (host clock around work that ends in a synchronise).  Synchronises the stream.
 * cfb_skeleton_read  the skeletons to the host, labels ascending (*num_labels <= num_objects entries of label_ids): label l has
 *     the vertices vertex_offsets[l] .. vertex_offsets[l + 1] (rows of float32 x, y, z at voxel centres, and radii) and the edges
 *     edge_offsets[l] .. edge_offsets[l + 1] (rows of two uint32 indices into its own vertices, sorted).  vertices and radii
 *     have num_skeleton_voxels rows, edges num_skeleton_voxels - num_objects; the offsets num_objects + 1 entries. */
int cfb_skeleton_workspace(int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes);
int cfb_edt_workspace(int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes);
int cfb_edt_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const double* voxel_size, float* d_dbf,
                   void* d_workspace, void* stream);
int cfb_skeleton_count_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const double* voxel_size,
                              const uint64_t* d_skip_ids, int64_t num_skip, int64_t dust_threshold, void* d_workspace, int64_t* num_objects,
                              int64_t* num_voxels, int64_t* buffer_bytes, void* stream);
int cfb_skeleton_device(const void* d_labels, int32_t dtype, int64_t z, int64_t y, int64_t x, const double* voxel_size, const double* params,
                        int32_t pdrf_exponent, void* d_workspace, int64_t num_objects, int64_t num_voxels, void* d_buffer,
                        int64_t buffer_bytes, int64_t* num_skeleton_voxels, double* stats, void* stream);
int cfb_skeleton_read(void* d_buffer, int64_t z, int64_t y, int64_t x, const double* voxel_size, int64_t num_objects, int64_t num_voxels,
                      int64_t num_skeleton_voxels, int64_t* num_labels, uint64_t* label_ids, int64_t* vertex_offsets, int64_t* edge_offsets,
                      float* vertices, uint32_t* edges, float* radii, void* stream);

/* `fill-segmentation-holes` (reference plugins/fill_segmentation_holes.py -> fill_voids.fill), rules restated in
 * oracle/fill_holes_oracle.py (fill_voids is not vendored: its 0/1 output is restated, not pinned; the hole mask equals
 * scipy.ndimage.binary_fill_holes(seg != 0)).  Connectivity 6 (face neighbours); "outside" is beyond the six faces of the
 * (z, y, x) chunk, which has fewer than 2^32 voxels.  An object is a 6-connected component of one non-zero id; object O encloses
 * voxel v (not in O) when every 6-connected path from v to outside passes through O.  The enclosers of a voxel are nested.
 *   CFB_FILL_BINARY           foreground = value != 0 (float32: -0 is background, NaN foreground); a hole is a background voxel
 *                             with no background path to outside.  Output 1 for foreground and holes, 0 elsewhere.  Count: the
 *                             holes.  dtype CFB_DTYPE_U8 (bool, uint8), CFB_DTYPE_F32, CFB_DTYPE_U32, CFB_DTYPE_U64.
 *   CFB_FILL_KEEP_ENCLOSED    every 0 voxel enclosed by an object takes the id of the innermost one; other voxels keep theirs.
 *                             Count: the enclosed zeros.
 *   CFB_FILL_REMOVE_ENCLOSED  every enclosed voxel, whatever its id, takes the id of the outermost encloser.  Count: every
 *                             enclosed voxel.  The per-object modes take CFB_DTYPE_U32 or CFB_DTYPE_U64 (signed ids by their
 *                             bit pattern).
 * Any other mode or dtype returns CFB_ERR_INVALID_ARGUMENT before any kernel runs; every error names its rule.
 * cfb_fill_holes_workspace        bytes of d_workspace (about 13 per voxel).  No device needed.
 * cfb_fill_holes_table_workspace  bytes of d_table for table_slots, a power of two below 2^31.  No device needed.
 * cfb_fill_holes_components_device  the 6-connected components (of the background in binary mode, of every value otherwise)
 *     and which of them reach outside, into d_workspace -> *num_components.  Synchronises the stream.
 * cfb_fill_holes_graph_device     (per-object modes) the distinct pairs of touching components into d_table -> *num_edges;
 *     CFB_ERR_CAPACITY when the table is too full -- call again with more slots.  Synchronises the stream.
 * cfb_fill_holes_enclose          (per-object modes) on the host: the innermost or outermost non-zero encloser of every component
 *     (articulation points of the component graph with a virtual outside node, iterative Hopcroft-Tarjan), written into
 *     d_workspace.  Synchronises the stream.
 * cfb_fill_holes_apply_device     d_out (same dtype and size as d_in, not overlapping it) = the filled chunk -> *fill_count.  After
 *     the components (binary) or the enclosure, with the same d_in.  Synchronises the stream. */
#define CFB_FILL_BINARY 0
#define CFB_FILL_KEEP_ENCLOSED 1
#define CFB_FILL_REMOVE_ENCLOSED 2
int cfb_fill_holes_workspace(int64_t z, int64_t y, int64_t x, int64_t* workspace_bytes);
int cfb_fill_holes_table_workspace(int64_t table_slots, int64_t* table_bytes);
int cfb_fill_holes_components_device(const void* d_in, int32_t dtype, int64_t z, int64_t y, int64_t x, int32_t mode, void* d_workspace,
                                     int64_t* num_components, void* stream);
int cfb_fill_holes_graph_device(void* d_workspace, int64_t z, int64_t y, int64_t x, void* d_table, int64_t table_slots, int64_t* num_edges,
                                void* stream);
int cfb_fill_holes_enclose(void* d_workspace, int64_t z, int64_t y, int64_t x, void* d_table, int64_t table_slots, int64_t num_edges,
                           void* stream);
int cfb_fill_holes_apply_device(const void* d_in, int32_t dtype, int64_t z, int64_t y, int64_t x, void* d_workspace, void* d_out,
                                int64_t* fill_count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CHUNKFLOW_B200_H_ */
