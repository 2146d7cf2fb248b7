/*
 * b200gen_metrics.h — the sample-quality metrics part of libb200gen.so's C-ABI: SSIM, MS-SSIM and MMD for judging
 * samples (generative/metrics of the reference), kept apart from b200gen.h, which describes the sampling path.
 */
#ifndef B200GEN_METRICS_H_
#define B200GEN_METRICS_H_

#include "b200gen.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Sample-quality metrics (generative/metrics/ssim.py, ms_ssim.py, mmd.py).  Inputs are planar tensors read in place
 * through element strides, in any of four formats; every value is converted to fp32 on load (the reference computes
 * in fp32 after convert_data_type(dtype=float)): B200_DT_F32, _F64, _FP16 and _BF16 of b200gen.h.
 * The conventions of b200gen.h hold (return codes, no allocation, no synchronisation, work enqueued on `stream`).
 * The ABI size query of b200gen.h answers 10 with sizeof(b200_ssim_params), 11 with sizeof(b200_ssim_combine_params).
 * The 2x average pooling between MS-SSIM scales is b200_interpolate's AREA mode over the even part of each extent.
 * ------------------------------------------------------------------------------------------------ */
#define B200_SSIM_MAX_K 128
#define B200_SSIM_MAX_SCALES 32

/* compute_ssim_and_cs (ssim.py:187-247) for one scale: x = y_pred, y = y, both [N][C][D][H][W] with element strides
 * {n, c, d, h, w} (2-D: D == 1, kd == 1).  The kernel is separable: taps_w[0..kw), taps_h[0..kh), taps_d[0..kd) (the
 * reference's fp32 gaussian_1d per axis, or all ones for the uniform kernel), and every filtered moment is multiplied
 * by `scale` once (the uniform kernel's fp32 1 / prod(kernel_size); 1 for the Gaussian).  Valid convolution: output
 * extents OD = D - kd + 1, OH = H - kh + 1, OW = W - kw + 1.  Per output voxel, in fp32:
 *   mu_* = scale * (filtered x, y, x*x, y*y, x*y)  (fused multiply-adds: W first, then H, then D, taps in order)
 *   sx = mu_xx - mu_x^2, sy = mu_yy - mu_y^2, sxy = mu_xy - mu_x mu_y
 *   cs = (2 sxy + c2) / (sx + sy + c2),  ssim = ((2 mu_x mu_y + c1) / (mu_x^2 + mu_y^2 + c1)) * cs
 * ssim_map / cs_map (NULL to skip) receive them as contiguous fp32 [N][C][OD][OH][OW].  Always: per CTA, the fp64 sums
 * of ssim and cs over its voxels go to `partials` (b200_ssim_workspace_bytes(p) bytes, [N][slots][2] doubles with
 * slots = bytes / (16 N)), which b200_ssim_combine reduces.  No atomics: two calls give identical bits.
 * Limits: kernel extents 1..B200_SSIM_MAX_K and no larger than the input; the tile (rows of x and y, the five W-filtered
 * moments and a ring of kd H-filtered planes) must fit in shared memory, which holds about k = 100 per axis in 3-D and
 * 120 in 2-D; larger kernels are B200_ENOTSUP.  The tile height (8, 4, 2 or 1 rows of 32 columns) is chosen from the
 * kernel size: the tallest that fits. */
typedef struct {
  const void* x;
  const void* y;
  int32_t x_dtype, y_dtype;            /* B200_DT_F32 / _F64 / _FP16 / _BF16 */
  int64_t x_strides[5], y_strides[5];  /* elements */
  int32_t N, C, D, H, W;
  int32_t kd, kh, kw;
  float taps_d[B200_SSIM_MAX_K], taps_h[B200_SSIM_MAX_K], taps_w[B200_SSIM_MAX_K];
  float scale, c1, c2;
  float* ssim_map;
  float* cs_map;
  double* partials;
} b200_ssim_params;
/* bytes of `partials` the call described by p writes (depends on the shapes and the device's SM count); -1 when the
 * call is invalid or its kernel does not fit.  Pointer fields are not read. */
int64_t b200_ssim_workspace_bytes(const b200_ssim_params* p);
int b200_ssim(const b200_ssim_params* p, void* stream);
/* Finish of SSIMMetric (ssim.py:135-139) and MultiScaleSSIMMetric (ms_ssim.py:134-151): per item n, per scale s,
 * mean_s = fp32(sum of partials[s] / count[s]) for ssim and cs (count = C * OD * OH * OW of that scale), written to
 * ssim_mean / cs_mean [n_scales][N] when not NULL; ms_ssim[n] (when not NULL) = prod_s relu(v_s) ** weights[s] in fp32,
 * v_s = cs mean of scale s, the ssim mean for the last scale.  One CTA per item; fixed summation order. */
typedef struct {
  const double* partials[B200_SSIM_MAX_SCALES];
  int32_t slots[B200_SSIM_MAX_SCALES];
  int64_t count[B200_SSIM_MAX_SCALES];
  float weights[B200_SSIM_MAX_SCALES];
  int32_t N, n_scales;
  float* ssim_mean;
  float* cs_mean;
  float* ms_ssim;
} b200_ssim_combine_params;
int b200_ssim_combine(const b200_ssim_combine_params* p, void* stream);
/* MMDMetric (mmd.py:36-70) with its linear kernel, beta = 1, gamma = 2: mean(Y Y^T) + mean(P P^T) - 2 mean(P Y^T) over
 * V = prod(shape[1..4]) equals sum_v (ybar_v - pbar_v)^2 / V, ybar and pbar the means over the batch, so one pass
 * reads each element once and no GEMM is formed.  y and y_pred are [shape[0]][shape[1]]..[shape[4]] with their own
 * element strides and dtypes; values are converted to fp32, their differences summed over the batch in fp64 and the
 * squares summed in fp64 per CTA (workspace: b200_mmd_workspace_bytes(shape) bytes); a second launch adds the CTA sums
 * in a fixed order and writes fp32(sum / (B^2 V)) to *out. */
int64_t b200_mmd_workspace_bytes(const int64_t* shape);
int b200_mmd(const void* y, int32_t y_dtype, const int64_t* y_strides, const void* y_pred, int32_t y_pred_dtype,
             const int64_t* y_pred_strides, const int64_t* shape, double* workspace, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GEN_METRICS_H_ */
