/*
 * b200gen_samplers.h — the multistep sampler step of libb200gen.so's C-ABI: one fused elementwise pass of
 * DPMSolverMultistepScheduler.step (DPM-Solver++, Lu et al. 2022, arXiv 2211.01095; orders 1-3 of the ODE form,
 * orders 1-2 of the SDE form).
 */
#ifndef B200GEN_SAMPLERS_H_
#define B200GEN_SAMPLERS_H_

#include "b200gen.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * The conventions of b200gen.h hold (return codes, no allocation, no synchronisation, work enqueued on `stream`).
 * b200_abi_sizeof(14) is sizeof(b200_dpm_coef).
 * ------------------------------------------------------------------------------------------------ */
#define B200_DPM_MAX_HIST 2

/* The solver's coefficients for one step, folded on the host in float64 and rounded once to fp32.  alpha_s, sigma_s
 * are sqrt(alphas_cumprod[s]) and sqrt(1 - alphas_cumprod[s]) of the current timestep s. */
typedef struct {
  float alpha_s, sigma_s;
  float c_x;                    /* weight of the sample                                      */
  float w[3];                   /* weights of x0 and of hist[0], hist[1] (earlier x0 estimates) */
  float c_z;                    /* weight of the noise (SDE form)                            */
  float clip_min, clip_max;
  int32_t prediction_type, clip;
} b200_dpm_coef;

/* b200_dpm_solver_step: over n fp32 elements, with s = sample, m = model_out, in fp32:
 *   x0 = (s - sigma_s * m) / alpha_s   (B200_PRED_EPSILON)
 *        alpha_s * s - sigma_s * m     (B200_PRED_V)
 *        m                             (B200_PRED_SAMPLE)
 *   x0 = min(max(x0, clip_min), clip_max)  if clip
 *   p  = c_x * s;  p = fma(w[0], x0, p);  p = fma(w[k + 1], hist[k], p) for k < n_hist;  p = fma(c_z, noise, p)
 *   prev_sample = p,  pred_x0 = x0.
 * hist is a host array of n_hist (0..B200_DPM_MAX_HIST) device pointers; noise may be NULL (no noise term).  Any
 * alignment; the outputs must not overlap the inputs. */
int b200_dpm_solver_step(const float* model_out, const float* sample, const float* const* hist, int32_t n_hist,
                         const float* noise, const b200_dpm_coef* c, float* prev_sample, float* pred_x0, int64_t n,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GEN_SAMPLERS_H_ */
