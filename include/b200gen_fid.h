/*
 * b200gen_fid.h — the Frechet Inception Distance part of libb200gen.so's C-ABI (FIDMetric of generative/metrics/fid.py
 * in the reference): fp64 feature moments and the Frechet distance between two Gaussians, kept apart from
 * b200gen_metrics.h (SSIM, MS-SSIM, MMD), whose fp32 conventions it does not share.
 */
#ifndef B200GEN_FID_H_
#define B200GEN_FID_H_

#include "b200gen.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 *   FID = |mu_x - mu_y|^2 + tr Sigma_x + tr Sigma_y - 2 tr sqrt(Sigma_x Sigma_y),  everything in fp64.
 * The conventions of b200gen.h hold (return codes, no allocation, no synchronisation, work enqueued on `stream`).
 * The ABI size query of b200gen.h answers 12 with sizeof(b200_fid_moments_params), 13 with
 * sizeof(b200_frechet_params).
 * ------------------------------------------------------------------------------------------------ */
#define B200_FID_MAX_F 32768

/* b200_fid_moments: one feature set x, [n][F] with element strides {row, feature} in any of the input formats
 * B200_DT_F32 / _F64 / _FP16 / _BF16 of b200gen.h, each value converted to fp64 exactly.  mu[f] = (sum of the n values
 * of feature f, rows in order within each of 16 interleaved partial sums, added in a fixed order) / n.
 * sigma = (X - mu)^T (X - mu) / (n - 1) as fp64(1 / (n - 1)) * Gram: mu is subtracted from every value on load and the
 * Gram is formed on the fp64 tensor cores; only the lower triangle's tiles are computed and each value is stored to
 * both triangles, so sigma is symmetric to the bit.  sigma is row-major [F][F].  Requires n >= 2 and
 * 1 <= F <= B200_FID_MAX_F.  No workspace. */
typedef struct {
  const void* x;
  int32_t x_dtype;           /* B200_DT_F32 / _F64 / _FP16 / _BF16 */
  int32_t F;
  int64_t n;
  int64_t x_strides[2];      /* elements: {row, feature} */
  double* mu;                /* [F] */
  double* sigma;             /* [F][F] */
} b200_fid_moments_params;
int b200_fid_moments(const b200_fid_moments_params* p, void* stream);

/* b200_frechet: the distance from (mu_x, sigma_x, mu_y, sigma_y), dense fp64, mu [F] and sigma row-major [F][F]
 * symmetric positive semidefinite (covariances).  Only the trace of the square root is formed: the nonzero eigenvalues
 * of Sigma_x Sigma_y are those of the symmetric M = G^T Sigma_x G for any G with Sigma_y = G G^T.
 *  1. Factor: pivoted Cholesky of Sigma_y by LAPACK dpstrf's rule, unblocked and right-looking.  At step j the pivot
 *     is the feature with the largest remaining (Schur-complement) diagonal entry among those not yet chosen; on a tie
 *     the lowest feature index wins.  The factorisation stops at rank r, at the first step whose maximum is
 *     <= F * 2^-52 * max(diag Sigma_y) (or is not a number); columns r..F-1 of G are exactly zero.  G = P L is kept
 *     in feature order: G[p_j][j] = sqrt(pivot), G[i][j] = W[p_j][i] / sqrt(pivot) for features i not yet chosen.
 *  2. M = G^T (Sigma_x G): two fp64 tensor-core GEMMs; the second computes the lower triangle's tiles and stores each
 *     value to both triangles, so M is symmetric to the bit.  Rows and columns r..F-1 of M are zero.
 *  3. Eigenvalues of M: Householder tridiagonalisation (unblocked, LAPACK dsytd2's reflectors), then bisection on
 *     Sturm counts from the Gershgorin interval, one thread per eigenvalue, at most 128 halvings.
 *  4. tr sqrt = sum of sqrt(mu_i) over eigenvalues mu_i > F * 2^-52 * mu_max, added in a fixed order; eigenvalues at
 *     or below that cutoff (the rounding-level ones a singular Sigma_x leaves) count as zero.
 * *out receives the distance.  eigvals (NULL to skip) receives the F eigenvalues of M in ascending order, rank (NULL to
 * skip) r.  Every loop has a fixed trip bound and nothing is added atomically: a non-finite value in the inputs gives
 * NaN in finite time, and two calls give identical bits.  About 2 launches per feature for the factor and 4 for the
 * tridiagonalisation, all stream-ordered.  workspace: b200_frechet_workspace_bytes(F) bytes (-1 when F is out of
 * range). */
typedef struct {
  const double* mu_x;
  const double* sigma_x;
  const double* mu_y;
  const double* sigma_y;
  int32_t F;
  int32_t reserved;          /* 0 */
  double* workspace;
  double* out;               /* 1 value */
  double* eigvals;           /* [F] or NULL */
  int32_t* rank;             /* 1 value or NULL */
} b200_frechet_params;
int64_t b200_frechet_workspace_bytes(int32_t F);
int b200_frechet(const b200_frechet_params* p, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GEN_FID_H_ */
