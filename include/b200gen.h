/*
 * b200gen.h — C-ABI of libb200gen.so: the sm_90a kernels behind the MONAI-GenerativeModels
 * diffusion *sampling* hot path (SURVEY.md §8).  Plain pointers and sizes only; no torch types.
 *
 * Conventions (SURVEY.md §8(b), inner boundary)
 *   - every entry point returns 0 on success or a negative B200_E* code; b200_last_error_string()
 *     gives the detail for the calling thread.  Nothing throws, exits, allocates device memory or
 *     synchronises the stream: all work is enqueued on `stream` (a cudaStream_t passed as void*).
 *   - activations are channels-last ("NDHWC") h16 unless a dtype field says otherwise; a 2-D image
 *     is D == 1; a token matrix [M, C] is D == H == 1, W == M.  The channel pitch of every h16
 *     activation is a multiple of 8 elements (16 bytes, the TMA global-stride granule).
 *   - each function cites the reference code (file:line under /root/reference) whose arithmetic it
 *     replaces.  The Python host (generativemodels_b200/) binds these with ctypes.
 */
#ifndef B200GEN_H_
#define B200GEN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK        0
#define B200_EINVAL   -1   /* bad shape / alignment / null pointer                    */
#define B200_ENOTSUP  -2   /* valid request this build has no kernel for              */
#define B200_ECUDA    -3   /* CUDA runtime / driver error, see b200_last_error_string */
#define B200_ENODEV   -4   /* device is not compute capability 9.0                    */

/* "h16" = the library's 16-bit storage type for activations and packed weights: IEEE fp16 in libb200gen.so (the
 * default: 11 significand bits, fp32 -> fp16 conversions saturate at +-65504), bfloat16 in the libb200gen_bf16.so
 * flavour built with -DB200_H16_IS_BF16.  b200_act_dtype() reports which one a loaded library computes in. */
#define B200_DT_H16  0
#define B200_DT_F32  1
/* input-only formats: b200_interpolate's x (on its one-element-per-thread path) and the metric inputs of
 * b200gen_metrics.h, converted to fp32 on load */
#define B200_DT_F64  2
#define B200_DT_FP16 3   /* IEEE half, whichever 16-bit format the library stores activations in */
#define B200_DT_BF16 4
#define B200_H16_FP16 0
#define B200_H16_BF16 1

#define B200_ACT_NONE 0
#define B200_ACT_RELU 1
#define B200_ACT_SILU 2
#define B200_ACT_GELU 4        /* exact erf GELU (nn.GELU default; monai MLPBlock act="GELU") */
#define B200_ACT_TANH 5        /* VQVAE output_act (vqvae.py:263-264, monai Act["TANH"])       */
#define B200_ACT_SIGMOID 6     /* VQVAE output_act (monai Act["SIGMOID"])                      */
#define B200_ACT_LEAKYRELU 3   /* nn.LeakyReLU() default slope 0.01 (monai act="LEAKYRELU" in blocks/spade_norm.py:52-60) */
/* b200_igemm act1 only: the GEGLU feed-forward of the transformer blocks (monai MLPBlock act="GEGLU",
 * diffusion_model_unet.py:211: linear1 -> a * gelu(gate) with a, gate = chunk(2, -1)) fused into linear1's epilogue.
 * The GEMM's `cout` columns come in 64-column groups [32 x a | 32 x gate] (the caller interleaves the weight rows and
 * the bias that way); output channel (col / 64) * 32 + col % 32 = (acc_a + bias_a) * gelu(acc_gate + bias_gate), so
 * the stored row has cout / 2 channels and no padding columns (out_cols == cout / 2).  Needs cout % 64 == 0, a h16
 * 16-byte-aligned output, no residual / scale / act2 / statistics / split. */
#define B200_ACT_GEGLU 7
/* nn.LeakyReLU(0.2): monai (act="LEAKYRELU", {"negative_slope": 0.2}), the default activation of SPADENet's encoder,
 * decoder output and residual blocks (nets/spade_network.py:82,158,245-246).  A code of its own rather than a slope
 * field, so that no parameter struct changes. */
#define B200_ACT_LEAKYRELU02 8

#define B200_IGEMM_MAX_SEG 128

const char* b200_last_error_string(void);
int b200_version(void);
/* B200_H16_FP16 or B200_H16_BF16: the 16-bit format this build stores activations / weights in. */
int b200_act_dtype(void);
/* 0 iff the current CUDA device is sm_90 (fails loudly elsewhere: there is no fallback). */
int b200_device_check(void);
int b200_sm_count(void);
/* sizeof() of the parameter structs below, for binding-layer ABI checks:
 * 0 igemm_params, 1 gn_stats_params, 2 gn_apply_params, 3 ddim_coef, 4 ddpm_coef, 5 pndm_coef, 6 igemm_seg,
 * 7 flash_params, 8 kl_coef, 9 repack_block. */
int b200_abi_sizeof(int which);

/* ------------------------------------------------------------------------------------------------
 * Implicit-GEMM on wgmma tensor cores (TMA-staged NDHWC tiles, accumulators in registers).
 * One kernel family serves every dense contraction on the path:
 *   - nn.Conv2d/3d k in {1,3,4}, stride {1,2}, symmetric or asymmetric zero padding
 *     (monai Convolution call sites: diffusion_model_unet.py:277,303,510,555,625,645,659,1748,1857;
 *      autoencoderkl.py:54-73,109,147-176; vqvae.py:61-77,127-162; controlnet.py:55-104,274-364)
 *   - nn.ConvTranspose k4 s2 p1 as one launch per output phase (vqvae.py:220-260)
 *   - channel-concat inputs read from two tensors (torch.cat at diffusion_model_unet.py:1232,1340,1461)
 *   - nn.Linear / q,k,v projections / GEGLU linears (diffusion_model_unet.py:98-103,211,379-381)
 *   - attention QK^T and PV as batched GEMMs (diffusion_model_unet.py:143-153,406-416)
 * out[n, od, oh, ow, co] = act2( residual + scale * act1( bias[co] + rowvec[n, co] + row_bias[ow] +
 *        sum_seg sum_c  A_src(seg)[n, od*sd + seg.dd, oh*sh + seg.dh, ow*sw + seg.dw, seg.c0*64 + c]
 *                        * W[wb, co, kbase(seg) + c] ) )
 * with out-of-range A coordinates / channels and W rows read as zero (TMA OOB fill).
 * kbase(seg) = 64 * (number of 64-channel chunks of all earlier segments).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int8_t  src;        /* which A tensor (0 or 1)                               */
  int8_t  dw, dh, dd; /* input offset of this tap, in input elements            */
  uint16_t c0;        /* first 64-channel chunk of the source read by this tap  */
  uint16_t nchunks;   /* number of 64-channel chunks                            */
} b200_igemm_seg;

typedef struct {
  /* A: up to two h16 NDHWC sources sharing N and the spatial extent */
  const void* a_ptr[2];
  int32_t a_C[2];      /* valid channels of each source                          */
  int32_t a_pitch[2];  /* elements between consecutive voxels (>= a_C, % 8 == 0) */
  int32_t in_N, in_D, in_H, in_W;
  int32_t stride_d, stride_h, stride_w;   /* conv stride (1 or 2)               */
  /* W: h16 [w_batch][w_rows][w_pitch], K-major, w_pitch % 64 == 0             */
  const void* w_ptr;
  int32_t w_rows;       /* valid rows (>= cout)                                  */
  int32_t w_pitch;      /* elements per row                                      */
  int32_t w_K;          /* valid K extent of a row (0 = w_pitch); reads past it are 0 */
  int64_t w_bstride;    /* elements between weight batches; 0 = shared weights   */
  int32_t w_batched;    /* 1: sample n uses weight batch n                       */
  int32_t n_seg;
  b200_igemm_seg seg[B200_IGEMM_MAX_SEG];
  /* output */
  void*   out_ptr;
  int32_t out_dtype;    /* B200_DT_H16 / B200_DT_F32                            */
  int32_t out_N, out_D, out_H, out_W;
  int32_t cout;         /* valid output channels                                 */
  int32_t out_cols;     /* channels stored per voxel (>= cout; extras get 0)     */
  int64_t out_sN, out_sD, out_sH, out_sW;   /* element strides; channel stride 1 */
  /* epilogue */
  const float* bias;    /* [cout] or NULL                                        */
  const float* rowvec;  /* [N or 1][rowvec_ld] fp32 per-sample vector or NULL    */
  int64_t rowvec_bstride; /* elements between samples (0 broadcasts)             */
  const float* row_bias; /* [out_W] fp32 added per output row (GEMM-shaped calls: out_D == out_H == 1) or NULL */
  int32_t act1;
  float   scale;        /* applied after act1                                    */
  const void* res_ptr;  /* residual, same logical shape as out, or NULL          */
  int32_t res_dtype;
  int64_t res_sN, res_sD, res_sH, res_sW;
  int32_t act2;
  float*  stat_ptr;     /* optional softmax partials: [out_W][ceil(out_cols/128)][2] = (max, sum exp(v - max)) over the
                           columns < cout of every 128-column tile of every output row, v = the fp32 value of `out`
                           above (after the residual and act2, before any 16-bit rounding); (-inf, 0) for a tile
                           with no such column.  GEMM-shaped calls only (out_N == out_D == out_H == 1), not with
                           impl = 1; NULL to skip                                                          */
  int32_t impl;         /* 0 = wgmma kernels (the planner picks one), 1 = CUDA-core cross-check kernel,
                           2 = the 128-column wgmma kernel only, 3 = the 128 x 256 two-CTA wgmma kernel
                           (B200_EINVAL for a call outside its envelope)                               */
  /* Optional GroupNorm partial sums for whoever normalises this output next (nn.GroupNorm after every conv of the
   * ResnetBlock, diffusion_model_unet.py:623-684): gn_partial[n][slot][cout/8][2] += (sum, sum of squares) of the
   * stored h16 values per 8-channel group; the kernel uses slots [gn_slot0, gn_slot0 + 4 * SM count) of the
   * gn_slots per sample, the caller zero-fills the buffer and b200_groupnorm_from_partials_ex reduces it.
   * Needs a h16, 16-byte-aligned output with cout % 32 == 0.  NULL to skip. */
  float*  gn_partial;
  int32_t gn_slots, gn_slot0;
  /* Optional split-K workspace.  A convolution on a small grid (the deep levels of a latent UNet: a few hundred
   * voxels x 20 000 reduction elements) has fewer output tiles than the GPU has SMs, and each tile walks its whole
   * reduction serially.  With a workspace of b200_igemm_split_workspace_bytes(p) bytes the reduction is cut into S
   * ranges computed by S CTAs per tile into fp32 partials [S][rows][round_up(out_cols, 8)], and a second kernel sums
   * them in a fixed order and applies the epilogue above (deterministic; fp32 summation order differs from the
   * unsplit kernel).  NULL / 0 = never split. */
  void*   split_ws;
  int64_t split_ws_bytes;
  /* 1: the A sources hold ONE sample that every one of the in_N samples reads (the operand-swapped projection
   * V^T[n] = W x[n]^T of a whole batch in one launch: A = the shared weight matrix, the per-sample activations are the
   * batched K-major operand, w_batched = 1).  0: sample n reads A at batch index n. */
  int32_t a_broadcast;
  /* Channels per gn_partial group: 8 (or 0 = 8; the layout described at gn_partial) or 4 — gn_partial[n][slot][cout/4][2],
   * for consumers whose GroupNorm groups are 4 channels wide (32 groups over 128 channels: level 0 of the 2-D UNets, the
   * AutoencoderKL). */
  int32_t gn_group;
} b200_igemm_params;

int b200_igemm(const b200_igemm_params* p, void* stream);
/* Host-only planning query, no CUDA call: what b200_igemm would choose for this call on a GPU with sm_count SMs —
 * out = {column tile (16..256), split factor (1 = one pass; > 1 only if with_workspace), work items, 0 (reserved)}.
 * The rules (DESIGN.md section 2): a convolution of >= 8 taps with a long reduction, 16-bit output and cout a multiple
 * of 256 whose units fill one wave of two-CTA clusters takes the 256-column kernel (work items = units of two M tiles);
 * otherwise, given a workspace, a call whose tiles fill at most half the SMs splits its reduction into
 * min(SMs / tiles, chunks of 64 / 32, 32) ranges when that is >= 3, and an unsplit call of >= 4 chunks halves its
 * column tile, down to 64, while the narrower tiles still fit one wave.  The rules are fixed: no setting changes them. */
int b200_igemm_plan(const b200_igemm_params* p, int32_t sm_count, int32_t with_workspace, int32_t out[4]);
/* Bytes of split_ws with which b200_igemm would split the reduction of this call; 0 when it would not (enough tiles
 * to fill the SMs, short reduction, stat_ptr / gn_partial requested, impl = 1).  Host-only, no launch. */
int64_t b200_igemm_split_workspace_bytes(const b200_igemm_params* p);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm (+SiLU) on NDHWC h16, optionally over the virtual concat of two tensors.
 * Replaces nn.GroupNorm + nn.SiLU in ResnetBlock / AttentionBlock / out head
 * (diffusion_model_unet.py:623-624,643,671,684, 372, 1853-1855; autoencoderkl.py:139-146,229).
 * Two phases: per-block partial sums -> per-(n,c) affine (a = fp32(rstd*gamma), b = fp32(beta - fp32(mean)*a)).
 * Statistics: the biased mean and variance of each group of the h16 inputs, rstd = 1 / sqrt(var + eps).  They are
 * summed as x - p with p the group's first element (channel g*C/groups at voxel 0), in fp32 per thread and folded in
 * fp64, so a large mean against the spread costs no precision: with s = sqrt(var + eps), the stats and fused
 * kernels give |d mean| <= 2^-12 (s + |mean - p|) and |d rstd| <= 2^-12 rstd (1 + (mean - p)^2 / s^2).
 * Only channels [0, x_C[i]) of the first N * spatial rows of each source are read (pad channels may hold anything).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const void* x_ptr[2];   /* h16 NDHWC sources (second may be NULL)      */
  int32_t x_C[2];         /* valid channels                               */
  int32_t x_pitch[2];     /* channel pitch                                */
  int32_t N;
  int64_t spatial;        /* D*H*W voxels per sample                      */
  int32_t groups;
  float   eps;
  const float* gamma;     /* [C0+C1]                                      */
  const float* beta;      /* [C0+C1]                                      */
  float*  partial;        /* workspace: b200_groupnorm_workspace_bytes()  */
  float*  affine;         /* out: [N][C0+C1][2] (a, b) fp32               */
} b200_gn_stats_params;
int64_t b200_groupnorm_workspace_bytes(int32_t N, int64_t spatial, int32_t C_total);
/* Writes affine [N][C0+C1][2] and nothing else but the workspace.  A group may straddle the two sources.  At most 6144
 * channels when every source is 16-byte aligned with C_i and x_pitch[i] multiples of 8 (the block reduction's shared
 * memory), at most 1024 otherwise; B200_EINVAL beyond. */
int b200_groupnorm_stats(const b200_gn_stats_params* p, void* stream);
/* The same affine table from partial sums that b200_igemm left while it wrote the tensor(s) (see gn_partial there),
 * so the statistics pass over the activations disappears.  group[i] is the producer group width of source i
 * (b200_igemm's gn_group: 8 or 4 channels per partial group; group NULL or an entry 0 = 8), and source i contributes
 * partial[i] = [N][slots[i]][x_C[i] / group[i]][2].  x_ptr of p is not read; every group of the virtual concat must be
 * a whole number of producer groups inside one source (C0 % ((C0+C1)/groups) == 0).  The fold is fp64 over the fp32
 * partials (mean = sum / n, var = sumsq / n - mean^2), exact to them up to fp64 rounding.  b200_igemm's partials are
 * raw fp32 sums of x and x^2, so unlike b200_groupnorm_stats this path loses rstd precision, about (mean / std)^2
 * 2^-24 times the terms per sum, when a group's mean is large against its spread. */
int b200_groupnorm_from_partials_ex(const b200_gn_stats_params* p, const float* const partial[2],
                                    const int32_t slots[2], const int32_t group[2], void* stream);

typedef struct {
  const void* x_ptr[2];
  int32_t x_C[2];
  int32_t x_pitch[2];
  int32_t N;
  int64_t spatial;
  const float* affine;    /* [N][C][2] from b200_groupnorm_stats          */
  int32_t act;            /* B200_ACT_NONE / SILU / LEAKYRELU / LEAKYRELU02 */
  void*   y_ptr;          /* h16 NDHWC, channel pitch y_pitch            */
  int32_t y_pitch;
} b200_gn_apply_params;
/* y = h16(act(fma(x, a, b))) per element (SiLU with __expf / __fdividef: a few fp32 ulps); pad channels [C, y_pitch)
 * of the N * spatial output rows are written +0, nothing past them.  Input pad channels are not read.  Another
 * activation (RELU, GELU, ...) is B200_EINVAL. */
int b200_groupnorm_apply(const b200_gn_apply_params* p, void* stream);

/* nn.GroupNorm (+ nn.SiLU) in ONE launch for small tensors (the deep levels of a latent UNet normalise 10^4..10^6
 * elements ~50 times per step: three launch latencies per GroupNorm for microseconds of work otherwise).  One CTA per
 * (sample, group) sums its slab, folds in fp64 and rewrites it; same arithmetic as stats + apply.  Reads x_ptr / x_C /
 * x_pitch / N / spatial / groups / eps / gamma / beta of `s` (partial and affine are not used) and act / y_ptr /
 * y_pitch of `a`.  With two sources no group may straddle them (C0 % (C / groups) == 0); at most 4096 channels per
 * group (and cpg / vec <= 512 for the widest vector vec in {8, 4, 2, 1} that channel counts, pitches and base
 * pointers allow), spatial < 2^24.  Meant for spatial * C / groups up to ~10^5 elements per group — larger tensors
 * want the two-phase form.  Statistics, output and footprint as stats + apply. */
int b200_groupnorm_fused(const b200_gn_stats_params* s, const b200_gn_apply_params* a, void* stream);

/* SPADE modulation (generative/networks/blocks/spade_norm.py:78-96), one pass:
 *   y = act( (x * ax + bx) * (1 + (g * ag + bg)) + (t * at + bt) )
 * x = virtual concat of the sources in p (GroupNorm affine table p->affine from b200_groupnorm_stats), g / t = the
 * gamma / beta halves of gb ([rows][gb_pitch] h16, channels [0,C) and [C,2C)) whose own per-(sample, channel)
 * InstanceNorm table gb_affine is [N][2C][2] (monai's Convolution default norm on mlp_gamma / mlp_beta).  Each factor
 * is one fp32 fma and the result h16(act(fma(nx, 1 + gg, tt))); gb_pitch >= 2C, and gb columns [2C, gb_pitch) and
 * input pad channels are not read; output pad channels [C, y_pitch) are written +0. */
int b200_spade_apply(const b200_gn_apply_params* p, const void* gb, int32_t gb_pitch, const float* gb_affine,
                     void* stream);

/* nn.LayerNorm over the last dim of a h16 [M, C] matrix (diffusion_model_unet.py:221-223): two fp32 passes (mean, then
 * the mean square of x - mean), one warp per row; with u = 2^-24 (C / 32 + 8) and s = sqrt(var + eps),
 * |d mean| <= u (|mean| + s) and |d rstd| <= rstd (u + 2^-21 + (d mean / s)^2).  Output h16((x - mean) rstd gamma +
 * beta), pad columns [C, y_pitch) +0; input columns [C, x_pitch) are not read. */
int b200_layernorm(const void* x, int64_t M, int32_t C, int32_t x_pitch, const float* gamma,
                   const float* beta, float eps, void* y, int32_t y_pitch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Layout / resampling / elementwise helpers on the API edge and between fused ops.
 * ---------------------------------------------------------------------------------------------- */
/* NC[D]HW fp32 -> NDHWC h16 (channel pitch `pitch`, pad channels zeroed; RN, fp16 saturates) and back (x_dtype
 * B200_DT_H16 or B200_DT_F32; input columns [C, pitch) are not read).  Both are exact apart from the one rounding. */
int b200_nchw_to_nhwc(const float* x, int32_t N, int32_t C, int64_t spatial, void* y, int32_t pitch,
                      void* stream);
int b200_nhwc_to_nchw(const void* x, int32_t x_dtype, int32_t N, int32_t C, int64_t spatial,
                      int32_t pitch, float* y, void* stream);
/* nn.Upsample(scale_factor=2, mode="bilinear" | "bicubic") on a 2-D NHWC h16 tensor [N][H][W][pitch] -> [N][2H][2W][pitch]
 * (SPADEDecoder's upsampling_mode, nets/spade_network.py:280,317), PyTorch's align_corners=False semantics: source
 * coordinate s = (dst + 0.5) / 2 - 0.5 per axis;
 *   B200_INTERP_BILINEAR: s clamped at 0, taps floor(s) and min(floor(s) + 1, in - 1) (the first even output: taps 0
 *                         and min(1, in - 1) with weights 1 and 0, as ATen computes it: an inf in row 0 stays inf, an
 *                         inf in row 1 makes it NaN);
 *   B200_INTERP_BICUBIC : s not clamped, taps floor(s) - 1 .. floor(s) + 2 each clamped to [0, in - 1], Keys cubic
 *                         convolution weights with A = -0.75 (upsample_bicubic2d), rows interpolated first.
 * At the fixed x2 scale the weights depend only on the output parity and are dyadic (0.25 / 0.75; Keys weights at
 * t = 0.25 / 0.75, at most 9 significant bits).  Arithmetic: along W within each source row an fp32 fma chain from 0
 * over the taps (each product exact, so one rounding per sum), then along H an fp32 fma chain from 0 over those rows;
 * one rounding on the store (fp16 saturates).  Every channel of the pitch is interpolated (zero pads stay zero).
 * pitch % 8 == 0, x and y 16-byte aligned. */
#define B200_INTERP_BILINEAR 0
#define B200_INTERP_BICUBIC  1
int b200_upsample2x_interp(const void* x, int32_t N, int32_t H, int32_t W, int32_t pitch, int32_t mode, void* y,
                           void* stream);
/* nn.AvgPool{2,3}d / nn.MaxPool{2,3}d(kernel_size=kernel, stride=2, padding=padding) on NDHWC h16 [N][D][H][W][pitch]
 * (MultiScalePatchDiscriminator's input pyramid, nets/patchgan_discriminator.py:89-92): dims == 2 pools H and W of
 * every D slice, dims == 3 all three.  Output extent per pooled axis floor((in + 2 * padding - kernel) / 2) + 1
 * (ceil_mode=False); requires 2 * padding <= kernel and in + 2 * padding >= kernel.
 *   B200_POOL_AVG: count_include_pad=True, i.e. the sum of the in-bounds taps divided by kernel^dims;
 *   B200_POOL_MAX: padding taps are -inf; a NaN tap makes the result NaN (PyTorch's max_pool semantics).
 * Arithmetic: avg sums the in-bounds taps in fp32 in d, h, w order from 0 (each partial sum rounded) and divides once
 * (IEEE) by kernel^dims; max is exact.  One rounding on the store (fp16 saturates).  Every channel of the pitch is
 * pooled (zero pads stay zero).  pitch % 8 == 0, x and y 16-byte aligned. */
#define B200_POOL_AVG 0
#define B200_POOL_MAX 1
int b200_pool_s2(const void* x, int32_t N, int32_t D, int32_t H, int32_t W, int32_t pitch, int32_t dims,
                 int32_t kernel, int32_t padding, int32_t mode, void* y, void* stream);
/* F.interpolate(x, size=... | scale_factor=..., mode=..., align_corners=False, antialias=False) at any size or scale
 * (SpatialRescaler, blocks/encoder_modules.py:60,78), and the library's other resampling on a grid: nearest x2
 * (diffusion_model_unet.py:578; autoencoderkl.py:84), nearest to a size (SPADE's segmentation map,
 * blocks/spade_norm.py:89), nn.AvgPool{2,3}d(2, 2) (diffusion_model_unet.py:522) and MS-SSIM's pooling between scales
 * (ms_ssim.py:130-131), the last two as AREA over the even part of each extent.  x is [N][C][D][H][W] and
 * y [N][C][OD][OH][OW] with arbitrary element strides {n, c, d, h, w} (host arrays x_strides / y_strides) and their own
 * dtypes (B200_DT_H16 / B200_DT_F32; x also B200_DT_F64 / _FP16 / _BF16, which only the one-element-per-thread path
 * below reads), so one entry point reads and writes planar NC[D]HW fp32, channels-last fp32 and channels-last h16.
 * `dims` is the number of resampled axes, the last ones: dims == 2 needs D == OD == 1, dims == 1 also H == OH == 1.
 * Modes and the dims they take (anything else is B200_EINVAL):
 *   B200_INTERPOLATE_NEAREST 1, 2, 3 | _LINEAR 1 | _BILINEAR 2 | _BICUBIC 2 | _TRILINEAR 3 | _AREA 1, 2, 3.
 * Coordinates follow ATen (ATen/native/UpSample.h and AdaptivePooling.h) per resampled axis, with the fp32 ratio r the
 * caller passes: r = float(1.0 / scale_factor) where F.interpolate was given a scale factor, else float(in) / out
 * (ATen's compute_scales_value: with an odd extent the two differ, e.g. 17 -> 8 samples 0.5, 2.5, ... with
 * scale_factor=0.5 but 0.5625, 2.6875, ... with size=8).  s = fma(r, dst + 0.5, -0.5) in fp32, one rounding, which is
 * ATen's r * (dst + 0.5) - 0.5 as its compilers contract it.
 *   NEAREST  : src = min(floor(dst * r), in - 1) (no identity shortcut: scale_factor=1.1 on 5 samples 0,0,1,2,3);
 *   linear family (LINEAR / BILINEAR / TRILINEAR): an axis with out == in is copied (its one tap dst read with weight
 *              1, so inf and NaN pass through);
 *              otherwise s is clamped at 0, i0 = min(floor(s), in - 1), i1 = i0 + (i0 < in - 1),
 *              l = clamp(s - i0, 0, 1), weights (1 - l, l);
 *   BICUBIC  : s not clamped, f = min(floor(s), in - 1), t = clamp(s - f, 0, 1), taps f - 1 .. f + 2 each clamped to
 *              [0, in - 1], Keys weights with A = -0.75: cc2(t + 1), cc1(t), cc1(1 - t), cc2(2 - t) where
 *              cc1(x) = ((A + 2) x - (A + 3)) x x + 1 and cc2(x) = ((A x - 5 A) x + 8 A) x - 4 A, each Horner step
 *              a fused multiply-add;
 *   AREA     : adaptive average pooling, window [floor(o * in / out), ceil((o + 1) * in / out)) per axis in integer
 *              arithmetic (the ratios are ignored).
 * Numerics: fp32 arithmetic, one rounding on the store (fp16 stores saturate).  NEAREST is a copy (bit-exact on finite
 * values when the dtypes match).  The separable modes interpolate along W within each source row first, then along H, then along D;
 * each 1-D step is sum_k x_k * w_k over its taps in order, products and sums rounded separately.  AREA sums the window
 * in d, h, w order (w innermost) and divides by the window's D, H and W extents in turn, as ATen does; on 2 x 2 (x 2)
 * windows that equals one scaling by 1/4 (1/8) except through double rounding when the mean is fp32-subnormal (a window
 * sum below 2^-124 in magnitude), which no fp16 input can give (every fp16 value is a multiple of 2^-24).
 * Threads: with channel stride 1 on both sides, every other stride a multiple of 8 elements, x and y 16-byte aligned
 * and w strides >= round_up(C, 8), one thread moves 8 channels as 16-byte vectors; these also write channels
 * [C, round_up(C, 8)) of every output voxel (a channels-last buffer's pad channels, interpolated from the input's
 * own: zeros stay zeros).  Otherwise one thread per output element, W fastest, so planar reads coalesce.
 * Extents up to 2^24 per axis (AREA: in * out + out <= 2^32); ratios of resampled axes positive and finite. */
#define B200_INTERPOLATE_NEAREST   0
#define B200_INTERPOLATE_LINEAR    1
#define B200_INTERPOLATE_BILINEAR  2
#define B200_INTERPOLATE_BICUBIC   3
#define B200_INTERPOLATE_TRILINEAR 4
#define B200_INTERPOLATE_AREA      5
int b200_interpolate(const void* x, int32_t x_dtype, const int64_t* x_strides, void* y, int32_t y_dtype,
                     const int64_t* y_strides, int32_t N, int32_t C, int32_t D, int32_t H, int32_t W, int32_t OD,
                     int32_t OH, int32_t OW, int32_t dims, int32_t mode, float ratio_d, float ratio_h, float ratio_w,
                     void* stream);
/* y = a + alpha * b on h16 buffers of n elements (ControlNet residual adds,
 * diffusion_model_unet.py:1917-1925,1931-1932; controlnet.py:405-407,433-434): h16(fma(alpha, b, a)) per element, over
 * all n elements (pad channels included: they must be finite).  n % 8 == 0; a, b and y 16-byte aligned. */
int b200_axpy_h16(const void* a, const void* b, float alpha, void* y, int64_t n, void* stream);
/* Copy C channels of every row of a channels-last h16 tensor into columns [dst_off, dst_off + C) of another
 * (materialises torch.cat([a, b], dim=1) only where a raw concatenated tensor is really needed).  The rest of each
 * destination row is left untouched; source columns [C, src_pitch) are not read. */
int b200_copy_channels(const void* src, int32_t C, int32_t src_pitch, void* dst, int32_t dst_pitch, int32_t dst_off,
                       int64_t rows, void* stream);
/* Tap reformulations for the degenerate convolutions at either end of the UNet (DiffusionModelUNet.conv_in with one
 * input channel, .out[2] with one output channel; diffusion_model_unet.py:1744-1752, 1856-1867).
 * geom = {N, D, H, W, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw} (input extent, output extent, kernel, stride,
 * low-side zero padding).
 * tap_gather: out[v][tap*C + c] = x[in_voxel(v, tap)][c] (zero outside the input), v over N*OD*OH*OW, h16 rows.
 * tap_sum:    out[v][co] = bias[co] + sum_tap y[v + off(tap)][tap*cout + co], y fp32 rows over the INPUT grid
 *             (stride 1, cout <= 4); out h16 or fp32, columns [cout, out_pitch) zeroed.
 * tap = (kd_i * kh + kh_i) * kw + kw_i.  tap_gather is a copy; it writes the whole row [0, out_pitch) (columns past
 * taps*C zero) and does not read x columns [C, x_pitch).  tap_sum adds in fp32 in tap order starting from the bias and
 * rounds once on an h16 store; y columns [taps*cout, y_pitch) are not read. */
int b200_tap_gather(const void* x, int32_t C, int32_t x_pitch, const int32_t* geom, void* out, int32_t out_pitch,
                    void* stream);
int b200_tap_sum(const float* y, int32_t y_pitch, const int32_t* geom, int32_t cout, const float* bias, void* out,
                 int32_t out_pitch, int32_t out_dtype, void* stream);
/* GEGLU: y[m, j] = x[m, j] * gelu_erf(x[m, H + j])  (monai MLPBlock act="GEGLU",
 * diffusion_model_unet.py:211). x: [M, 2H] pitch x_pitch; y: [M, H] pitch y_pitch.  fp32 with erff, one rounding on
 * the store.  Columns [H, y_pitch) of y are not written, columns [2H, x_pitch) of x not read.  M >= 1, H, x_pitch and
 * y_pitch multiples of 8 (H >= 8), x and y 16-byte aligned. */
int b200_geglu(const void* x, int64_t M, int32_t H, int32_t x_pitch, void* y, int32_t y_pitch,
               void* stream);
/* softmax over rows of an fp32 [M, S] score matrix -> h16 probabilities [M, p_pitch]
 * (attention_scores.softmax(dim=-1), diffusion_model_unet.py:150,412) in ONE pass over the scores: the row maximum and
 * sum come from the per-(row, 128-column tile) partials b200_igemm wrote (stat_ptr), n_tiles per row.
 * p = h16(exp(s - max) * (1 / sum)), normalised in fp32 before the one rounding.  Pad columns [S, p_pitch) are
 * written +0; rows past M are not written. */
int b200_softmax_rows_partials(const float* s, int64_t M, int32_t S, int64_t s_pitch, const float* partials,
                               int32_t n_tiles, void* p, int64_t p_pitch, void* stream);

/* Flash-style attention on wgmma (scores stay in registers; online softmax; head_dim in {64,128,256,512}, any T, S).
 * q: [B][T][q_pitch], k: [B][S][k_pitch] h16 rows with heads as channel slices [h*dh, (h+1)*dh);
 * vt: V transposed, [B][heads*dh][vt_pitch] (key index contiguous); out / res: [B][T][pitch] h16; res may be NULL.
 * out[b,t,h*dh+c] = sum_s softmax_s(scale * q.k)[s] * v[s,c] (+ res).   (diffusion_model_unet.py:143-153, 406-416)
 * Numerics: sigma_s = fp32(scale * log2 e) * q.k in fp32; the running row maximum m advances once per key block (64
 * keys; 128 for head_dim 512); each probability is rounded to h16 from fp32 as P~_s = h16(2^(sigma_s - m_block(s)))
 * (ex2.approx.ftz), the denominator l = sum_s 2^(sigma_s - m) is accumulated in fp32 from the unrounded values, and
 * out = h16(sum_s P~_s 2^(m_block(s) - m) v_s / l + res) with the residual added in fp32 before the one rounding.
 * Only [B][T][heads*dh] of out is written: not the pad columns [heads*dh, out_pitch), not rows past T.  Not read:
 * q / k columns past heads*dh, V^T columns [S, vt_pitch), residual columns past heads*dh.
 * B200_EINVAL for another head_dim, a pitch (res_pitch with res) not a multiple of 8, a pointer not 16-byte aligned,
 * or B, T, S, heads < 1.  (tests/test_attention_contract_gpu.py checks all of this against tests/attention_emulator.py.) */
typedef struct {
  const void* q; const void* k; const void* vt; void* out; const void* res;
  int32_t B, T, S, heads, dh;
  int32_t q_pitch, k_pitch, vt_pitch, out_pitch, res_pitch;
  float scale;
  /* Reserved scratch: the kernel keeps every probability tile on chip and needs none
   * (b200_attention_flash_workspace_bytes() returns 0); both fields are ignored. */
  void* workspace; int64_t workspace_bytes;
} b200_flash_params;
int b200_attention_flash(const b200_flash_params* p, void* stream);
/* bytes of scratch the call described by p can use (0 when none is needed); pointer fields are not read */
int64_t b200_attention_flash_workspace_bytes(const b200_flash_params* p);

/* Small-shape attention on CUDA cores (any head_dim <= 1024, any S); used for the test-suite
 * head dims (2..8), for head dims that are not multiples of 64 and for cross-attention with a handful of context tokens.
 * q: [B, T, H*dh] h16 pitch q_pitch; k, v: [B, S, H*dh]; out: [B, T, H*dh].  Pitches need no alignment.
 * fp32 scores, online softmax and accumulation; only the output is rounded, and only its [B][T][H*dh] is written.
 * (CrossAttention._attention, diffusion_model_unet.py:136-153; AttentionBlock 406-416.) */
int b200_attention_small(const void* q, const void* k, const void* v, void* out, int32_t B, int32_t T,
                         int32_t S, int32_t heads, int32_t dh, int32_t q_pitch, int32_t k_pitch,
                         int32_t v_pitch, int32_t o_pitch, float scale, void* stream);
/* The same with the two things the autoregressive transformer needs (blocks/selfattention.py:93-140,
 * inferer.py:1183-1245): k / v may live in a cache of kv_rows >= S rows per batch item, and with causal != 0 query
 * row t (absolute position q_pos0 + t) attends to keys s <= q_pos0 + t only.  With pos_dev != NULL the prefix length
 * is read on the device (q_pos0 = *pos_dev, S = *pos_dev + T): the decode step can then be captured ONCE in a CUDA
 * graph and replayed for every token. */
int b200_attention_small_ex(const void* q, const void* k, const void* v, void* out, int32_t B, int32_t T,
                            int32_t S, int32_t heads, int32_t dh, int32_t q_pitch, int32_t k_pitch,
                            int32_t v_pitch, int32_t o_pitch, float scale, int32_t kv_rows, int32_t causal,
                            int32_t q_pos0, const int32_t* pos_dev, void* stream);
/* Token + absolute position embedding rows (nets/transformer.py:20-37, 97-99):
 * out[m, :] = tok_emb[tokens[m], :] + pos_emb[pos0 + m % seq_len, :], h16 rows of pitch `pitch`
 * (pos0 = *pos_dev when pos_dev != NULL): one fp32 add, one rounding; pad columns [C, pitch) +0.  Precondition, not
 * checked: every token id indexes a row of tok_emb and every pos0 + m % seq_len a row of pos_emb. */
int b200_embed_tokens(const int64_t* tokens, int64_t M, int32_t seq_len, int32_t pos0, const float* tok_emb,
                      const float* pos_emb, int32_t C, void* out, int32_t pitch, const int32_t* pos_dev, void* stream);
/* Graph-captured decoding: append T rows per sequence to a [B, L, pitch] h16 cache at the device-side position,
 * and advance that position.  cache[b][pos + t] = src[b * T + t] (a copy); rows with pos + t outside [0, L) are dropped. */
int b200_cache_append(const void* src, void* cache, int32_t B, int32_t T, int32_t L, int32_t pitch,
                      const int32_t* pos_dev, void* stream);
int b200_advance_i32(int32_t* p, int32_t delta, void* stream);
/* Decode-time linear layers (one new token per sequence: M <= 8 rows, HBM/L2-bound GEMVs):
 *   out[m, o] = act( LN?(x[m, :]) . w[o, :K] + bias[o] ) + res[m, o]
 * x h16 rows; ln_gamma / ln_beta (NULL = no LayerNorm; nn.LayerNorm semantics with b200_layernorm's arithmetic and
 * accuracy, the row rounded to h16 as the stand-alone kernel does); w = the K-major h16 matrix b200_igemm consumes (row
 * pitch w_pitch, a multiple of 8 and >= round_up(K, 8), 16-byte aligned); bias fp32 or NULL; res h16 or NULL; out h16 or
 * fp32 (out_dtype).  Arithmetic: each of a warp's 32 lanes sums 8 columns of every 256 in an fp32 fma chain
 * (8 ceil(K / 256) terms), a 5-level butterfly folds the lanes, then the bias add, act (b200_small_linear's), the
 * residual add in fp32 and one rounding on an h16 store (fp16 saturates).  Not read: x columns [K, x_pitch), w columns
 * [K, w_pitch), res columns [O, r_pitch).  Not written: out columns [O, o_pitch).  B200_EINVAL for M outside 1..8,
 * M * round_up(K, 8) * 2 > 48 KB, or a pitch below its row.  (blocks/transformerblock.py:87-92,
 * blocks/selfattention.py:103-110, 145.) */
int b200_rows_linear(const void* x, int32_t x_pitch, int32_t M, int32_t K, const float* ln_gamma,
                     const float* ln_beta, float ln_eps, const void* w, int32_t w_pitch, int32_t O, const float* bias,
                     int32_t act, const void* res, int32_t r_pitch, void* out, int32_t o_pitch, int32_t out_dtype,
                     void* stream);
/* One query row per (batch, head) against S cached keys / values ([B, kv_rows, pitch] h16; S = *pos_dev + 1 when
 * pos_dev != NULL): the keys are split over the warps of a block and the online-softmax states merged (warps without
 * a key count nothing).  head_dim <= 256; fp32 throughout, only the output [B][heads*dh] rounded and written. */
int b200_attention_decode(const void* q, const void* k, const void* v, void* out, int32_t B, int32_t S,
                          int32_t heads, int32_t dh, int32_t q_pitch, int32_t k_pitch, int32_t v_pitch,
                          int32_t o_pitch, float scale, int32_t kv_rows, const int32_t* pos_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Time embedding path (diffusion_model_unet.py:461-485, 1759-1767, 1888-1902; ResnetBlock 641,686).
 * ---------------------------------------------------------------------------------------------- */
/* emb[n, :] = [cos(t_n f_i) ..., sin(t_n f_i) ...], f_i = exp(-ln(max_period) i / half), zero-pad if odd
 * (half = dim / 2; dim == 1 is all zeros).  fp32 logf / expf / cosf / sinf.  N * dim < 2^31. */
int b200_timestep_embedding(const float* t, int32_t N, int32_t dim, float max_period, float* emb,
                            void* stream);
/* y[m, o] = act_out( b[o] + sum_k act_in(x[m, k]) W[o, k] ), fp32 (GEMV-class: one warp per output feature loops over
 * the rows; 1 <= M <= 4096).  b may be NULL.  Each lane sums its k in an fp32 fma chain, the lanes fold in a warp tree. */
int b200_small_linear(const float* x, int32_t M, int32_t K, const float* W, const float* b, int32_t O,
                      int32_t act_in, int32_t act_out, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Scheduler steps: one fused elementwise pass each (fp32 tensors of n elements).
 * ---------------------------------------------------------------------------------------------- */
#define B200_PRED_EPSILON  0
#define B200_PRED_SAMPLE   1
#define B200_PRED_V        2
/* DDIMScheduler.step (ddim.py:156-237): coefficients computed on the host exactly as the reference
 * does (0-dim fp32 tensor arithmetic) and passed by value. noise may be NULL (eta == 0). */
typedef struct {
  float sqrt_alpha_prod_t, sqrt_beta_prod_t;   /* alpha_prod_t**0.5, beta_prod_t**0.5            */
  float sqrt_alpha_prod_prev, dir_coef;        /* alpha_prod_t_prev**0.5, (1-a_prev-var)**0.5    */
  float sigma;                                 /* eta * variance**0.5                            */
  float clip_min, clip_max;                    /* clip_sample_values (ddim.py:213-216)           */
  int32_t prediction_type, clip;
} b200_ddim_coef;
int b200_ddim_step(const float* model_out, const float* sample, const float* noise,
                   const b200_ddim_coef* c, float* prev_sample, float* pred_x0, int64_t n, void* stream);
/* DDPMScheduler.step (ddpm.py:191-252): mean = c_x0 * clamp(x0) + c_xt * x_t, + sigma * noise. */
typedef struct {
  float sqrt_alpha_prod_t, sqrt_beta_prod_t;
  float coef_x0, coef_xt;      /* pred_original_sample_coeff, current_sample_coeff (ddpm.py:235-236) */
  float sigma;                 /* variance ** 0.5 for the fixed variance types (ddpm.py:158-189)     */
  float clip_min, clip_max;
  float min_log, max_log;      /* learned_range: variance = frac*max_log + (1-frac)*min_log          */
  int32_t var_mode;            /* 0 fixed (sigma), 1 learned (pred_var), 2 learned_range             */
  int32_t prediction_type, clip;
} b200_ddpm_coef;
/* noise == NULL at t == 0 (no noise is added, ddpm.py:243); pred_var only for learned variance. */
int b200_ddpm_step(const float* model_out, const float* sample, const float* noise, const float* pred_var,
                   const b200_ddpm_coef* c, float* prev_sample, float* pred_x0, int64_t n, void* stream);
/* One timestep of DiffusionInferer.get_likelihood (inferer.py:205-265, 279-321), fused: from x_0 (inputs), x_t
 * (noisy) and the model output compute the predicted and posterior means, then the per-element KL between the two
 * normals (t > 0) or the discretised-Gaussian decoder negative log-likelihood (t == 0); kl_out (optional) receives
 * the per-element fp32 term, sample_sum[n] += the fp64 sum of those fp32 terms over the sample's elements.  The
 * summation order is unspecified (fp64 atomics across CTAs), so sample_sum can differ between calls in its last bits.
 * Fixed-variance schedulers. */
typedef struct {
  float sqrt_alpha_prod_t, sqrt_beta_prod_t;
  float coef_x0, coef_xt;              /* shared by the predicted mean (ddpm.py:235-240) and _get_mean (133-156)   */
  float log_pred_var, log_post_var;    /* log of the (fixed) predicted / posterior variance                        */
  float bin_width;                     /* (scaled range) / (original range), decoder term only                     */
  int32_t prediction_type, clip, is_t0;
} b200_kl_coef;
int b200_ddpm_kl(const float* x0, const float* xt, const float* model_out, const b200_kl_coef* c, float* kl_out,
                 double* sample_sum, int32_t N, int64_t per_sample, void* stream);
/* PNDMScheduler._get_prev_sample after the linear-multistep combine (pndm.py:261-273, 293-315):
 * eps = sum_i w[i] * hist[i] (up to 4 history tensors), prev = sample_coeff*sample - eps_coeff*eps.
 * eps_out (optional) receives the combined model output; prev_sample may be NULL (PRK accumulation,
 * pndm.py:204-224). v-prediction pre-mix per pndm.py:304-305. */
typedef struct {
  float w[4];
  int32_t n_hist;
  float sample_coeff, eps_coeff;
  float v_alpha, v_beta;  /* alpha_prod_t**0.5, beta_prod_t**0.5 for v-prediction */
  int32_t prediction_type;
} b200_pndm_coef;
int b200_pndm_step(const float* const* hist, const float* sample, const b200_pndm_coef* c,
                   float* prev_sample, float* eps_out, int64_t n, void* stream);
/* AutoencoderKL.encode tail (autoencoderkl.py:731-734): sigma = exp(clamp(log_var, lo, hi) / 2), fp32. */
int b200_exp_half_clamped(const float* log_var, float lo, float hi, float* sigma, int64_t n, void* stream);
/* SPADENet's VAE step (nets/spade_network.py:214-217, 33-34) over n fp32 elements:
 *   z[i] = eps[i] * exp(0.5 * logvar[i]) + mu[i],   kld[0] = -0.5 * sum_i (1 + logvar[i] - mu[i]^2 - exp(logvar[i])).
 * eps is drawn by the caller.  One CTA sums in a fixed order (fp64), so kld is the same on every call. */
int b200_vae_reparam_kld(const float* mu, const float* logvar, const float* eps, float* z, float* kld, int64_t n,
                         void* stream);
/* out = x * mul / div, fp32 (latent scale_factor handling, inferer.py:385, 472-475). */
int b200_scale_f32(const float* x, float mul, float div, float* out, int64_t n, void* stream);
/* AutoencoderKL.sampling (autoencoderkl.py:751-752): out = a + b * c elementwise, fp32. */
int b200_fma_f32(const float* a, const float* b, const float* c, float* out, int64_t n, void* stream);
/* Scheduler.add_noise / get_velocity (scheduler.py:169-200) with per-sample coefficients. */
int b200_add_noise(const float* x0, const float* noise, const float* ca, const float* cb, float sign_b,
                   int32_t N, int64_t per_sample, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Vector quantiser (vector_quantizer.py:86-138): nearest codebook row under
 * d = |x|^2 + |e|^2 - 2 x.e (fp32), first index wins ties; writes int64 indices and optionally the
 * gathered rows.  x: fp32 [M, D] (channels-last, row pitch x_pitch; columns [D, x_pitch) not read); codebook fp32 [K, D].
 * Order: |x|^2, |e|^2 and x.e are each one fma chain over d = 0 .. D-1 from 0, then d = (|x|^2 + |e|^2) - 2 x.e.
 * A row whose distances are all NaN (or +inf) gets index 0.  sqerr_sum is added to with fp64 atomics (order
 * unspecified).  D == 32 takes a register-tiled kernel with the same arithmetic (bit-identical indices).
 * ---------------------------------------------------------------------------------------------- */
/* Optional outputs (NULL to skip): q_h16 rows (pitch q_pitch, pad zeroed) for the decoder; q_f32 [M, D] with the
 * straight-through rounding x + (q - x) when ste != 0 (vector_quantizer.py:186) else q; sqerr_sum += sum (q-x)^2
 * (commitment loss numerator, 183); hist[k] += count (perplexity, 212-218). */
int b200_vq_argmin_gather(const float* x, int64_t M, int32_t D, int32_t x_pitch, const float* codebook,
                          int32_t K, int64_t* indices, void* q_h16, int32_t q_pitch, float* q_f32,
                          int32_t ste, double* sqerr_sum, int32_t* hist, void* stream);
/* nn.Embedding gather for decode_samples (vqvae.py:445-450): idx int64 [M] -> h16 rows (pad columns +0).  Indices
 * outside [0, K - 1] are clamped into it. */
int b200_vq_gather(const int64_t* indices, int64_t M, const float* codebook, int32_t K, int32_t D,
                   void* q_h16, int32_t q_pitch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Weight repacking (SURVEY.md section 8b: b200_repack_conv_weight / b200_repack_linear_weight): one launch turns an fp32
 * parameter into the K-major h16 matrix [rows_pad][dst_pitch] that b200_igemm's weight tensor map reads.  The matrix
 * is a sequence of column BLOCKS, one per b200_igemm segment (filter tap x input-tensor split), each ceil64(cs) wide:
 *   dst[co][blk.col0 + c] = sum_{t < blk.ntaps} src(co, blk.cin0 + c, blk.tap[t])      for c < blk.cs, co < cout
 * and zero elsewhere (channel tails, pad rows).  Plain convolutions have one source tap per block; the nearest-x2
 * upsample folded into a 3^d convolution (diffusion_model_unet.py:574-586) sums up to 8 original taps per phase tap
 * (added in index order, fp32); a transposed convolution (vqvae.py:220-260) packs the taps of one output phase.
 *   src layout: transposed == 0: [cout][cin][taps] (nn.ConvNd / nn.Linear with taps == 1);
 *               transposed == 1: [cin][cout][taps] (nn.ConvTransposeNd).
 * mode B200_REPACK_TAP_IN  : dst[co][tap * cin + c] = src[co][c][tap]   (few-input-channel convs as ONE K chunk)
 * mode B200_REPACK_TAP_OUT : dst[tap * cout + co][c] = src[co][c][tap]   (few-output-channel convs: taps as GEMM rows)
 * `blocks` is a HOST array (copied into the launch parameters; at most B200_IGEMM_MAX_SEG entries).
 * ---------------------------------------------------------------------------------------------- */
#define B200_REPACK_BLOCKS  0
#define B200_REPACK_TAP_IN  1
#define B200_REPACK_TAP_OUT 2
typedef struct {
  int32_t col0;       /* first destination column (multiple of 64)     */
  int32_t cin0, cs;   /* source channel range [cin0, cin0 + cs)         */
  int32_t ntaps;      /* 1..8 source taps summed into this block        */
  int16_t tap[8];     /* flattened source tap indices                   */
} b200_repack_block;
int b200_repack_weight(const float* src, int32_t cout, int32_t cin, int32_t taps, int32_t transposed, int32_t mode,
                       const b200_repack_block* blocks, int32_t n_blocks, void* dst, int32_t rows_pad,
                       int32_t dst_pitch, void* stream);
/* Eval-mode nn.BatchNorm{2,3}d folded into the convolution that feeds it (monai Convolution with ADN order "NDA" and
 * norm="BATCH", PatchDiscriminator's hidden layers, nets/patchgan_discriminator.py:229-240), before
 * b200_repack_weight rounds the result to h16 once:
 *   s[co] = gamma[co] / sqrt(var[co] + eps)
 *   w_out[co][j] = w[co][j] * s[co]                       for j < per_out (= cin * taps, the parameter's layout)
 *   b_out[co]    = beta[co] + (b[co] - mean[co]) * s[co]  (b == NULL: a convolution without bias, b = 0)
 * IEEE fp64 arithmetic (division, square root, multiplication), one rounding to fp32 per output: w_out is exact to
 * that; b_out's multiply-add may be contracted into a double fma, which can move it to the neighbouring fp32 value.
 * All arrays fp32 device memory.  B200_EINVAL for a NULL array other than b, cout or per_out < 1, or eps < 0. */
int b200_batchnorm_fold(const float* w, const float* b, const float* gamma, const float* beta, const float* mean,
                        const float* var, float eps, int32_t cout, int64_t per_out, float* w_out, float* b_out,
                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GEN_H_ */
