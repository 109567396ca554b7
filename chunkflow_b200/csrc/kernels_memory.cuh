// HBM-bound kernels of the inference hot path: patch extract (+u8 normalise), bump-mask
// blend, weight-volume gather, final normalise, identity backend.  Declarations.
#pragma once
#include "common.cuh"

namespace cfb {

// a6+a7 (reference inferencer.py:395-399,409-411; chunk/base.py:761-781): cut `nb`
// patches out of the chunk into (nb,1,pz,py,px) fp32; uint8 input is normalised with a
// true division by 255 (bit-identical to numpy's astype(float32) / 255).
void launch_extract_patches(const void* chunk, int in_dtype, Int3 chunk_size, const PatchPos* patches,
                            int nb, Int3 patch, float* out, cudaStream_t s);

// a9-tail + a11 (reference patch/pytorch.py:112-113, chunk/base.py:792-807): crop the
// network output, multiply by the bump mask and accumulate into the output chunk.
// net: (nb, cnet, pz,py,px) fp32; mask: (oz,oy,ox) fp32 of the output patch; out: (C, OZ,OY,OX).
void launch_blend_patches(const float* net, int cnet, Int3 in_patch, Int3 out_patch, Int3 crop,
                          const float* mask, const PatchPos* patches, int nb, float* out, int channels,
                          Int3 out_size, float scale, cudaStream_t s);

// identity backend (reference patch/identity.py:30-51) fused with extract and blend.
void launch_identity_blend(const void* chunk, int in_dtype, Int3 chunk_size, Int3 in_patch, Int3 out_patch,
                           Int3 crop, const float* mask, const PatchPos* patches, int nb, float* out,
                           int channels, Int3 out_size, cudaStream_t s);

// plugin level (reference patch/pytorch.py:112-113, patch/identity.py:41-49): crop + mask of
// `nb` network outputs into a dense (nb, channels, oz,oy,ox) array; `repeat` broadcasts
// source channel 0 to every output channel (identity backend's np.repeat).
void launch_crop_mask(const float* net, int cnet, Int3 in_patch, Int3 out_patch, Int3 crop, const float* mask,
                      int nb, float* out, int channels, bool repeat, cudaStream_t s);

// Device tables of the weight-volume gather: per output axis, the cover table (kMaxCover patch axis-indices per
// coordinate) and the output start of every patch axis-index.
struct CoverTables {
  const int *cover_z, *cover_y, *cover_x;
  const int *ostart_z, *ostart_y, *ostart_x;
};

// a5 (reference inferencer.py:294-333): W(v) = sum over covering patches (in patch-list
// order) of mask(v - o_p); writes 1/W if `invert`, else W.
void launch_weight_volume(const float* mask, Int3 out_patch, const CoverTables& t, Int3 out_size, float* w, bool invert,
                          cudaStream_t s, int z_begin = 0, int z_end = -1);

// dst[i] += src[i]: halo planes received from another rank (one chunk split over GPUs, BASELINE config #5).
void launch_halo_add(float* dst, const float* src, int64_t n, cudaStream_t s);

// a12+a13 (reference inferencer.py:460-466): out *= winv (broadcast over channels), and
// track the maximum into *max_bits (float bits, values are >= 0).  If *zero_flag == 0
// (all-zero input, reference :387-393) the output is forced to zero.
// `nvox` voxels per channel starting at `out` / `winv`; channels are `channel_stride` floats apart
// (0 = nvox), so a z-range of planes of a larger volume can be normalised on its own.
void launch_normalize(float* out, const float* winv, bool w_is_inverse, int channels, int64_t nvox,
                      unsigned int* max_bits, const unsigned int* nonzero_flag, cudaStream_t s,
                      int64_t channel_stride = 0);

// a14 (reference chunk/base.py:685-689): out[c] *= (out[last] < thr) for c < channels-1.
void launch_myelin_mask(float* out, int channels, int64_t nvox, float threshold, cudaStream_t s);

// all-zero test of the input chunk (reference inferencer.py:387): sets *flag to 1 if any
// byte/value is non-zero.
void launch_any_nonzero(const void* chunk, int in_dtype, int64_t n, unsigned int* flag, cudaStream_t s);

}  // namespace cfb
