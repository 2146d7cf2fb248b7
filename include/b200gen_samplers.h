/*
 * b200gen_samplers.h — the multistep sampler steps of libb200gen.so's C-ABI: one fused elementwise pass of
 * DPMSolverMultistepScheduler.step (DPM-Solver++, Lu et al. 2022, arXiv 2211.01095; orders 1-3 of the ODE form,
 * orders 1-2 of the SDE form) and one of UniPCMultistepScheduler.step (UniPC, Zhao et al. 2023, arXiv 2302.04867;
 * the data-prediction form, predictor orders 1-3 with the UniC corrector) and one of SASolverScheduler.step
 * (SA-Solver, Xue et al. 2023, arXiv 2309.05019; the data-prediction form of the stochastic Adams predictor-corrector).
 */
#ifndef B200GEN_SAMPLERS_H_
#define B200GEN_SAMPLERS_H_

#include "b200gen.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * The conventions of b200gen.h hold (return codes, no allocation, no synchronisation, work enqueued on `stream`).
 * b200_abi_sizeof(14) is sizeof(b200_dpm_coef), b200_abi_sizeof(15) is sizeof(b200_unipc_coef),
 * b200_abi_sizeof(16) is sizeof(b200_sa_solver_coef).
 * ------------------------------------------------------------------------------------------------ */
#define B200_DPM_MAX_HIST 2
#define B200_UNIPC_MAX_HIST 3
#define B200_SA_SOLVER_MAX_HIST 2

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

/* UniPC's corrector and predictor for one step, each folded on the host in float64 and rounded once to fp32. */
typedef struct {
  float alpha_s, sigma_s;       /* of the current timestep, to form x0 as in b200_dpm_solver_step                */
  float c_last;                 /* corrector: weight of the previous step's corrected sample                     */
  float v[4];                   /* corrector: weights of x0 and of hist[0], hist[1], hist[2]                     */
  float c_xc;                   /* predictor: weight of the corrected sample                                     */
  float u[3];                   /* predictor: weights of x0 and of hist[0], hist[1]                              */
  float clip_min, clip_max;
  int32_t prediction_type, clip;
} b200_unipc_coef;

/* b200_unipc_step: over n fp32 elements, with s = sample, m = model_out, in fp32:
 *   x0 as in b200_dpm_solver_step (prediction type, then the clip)
 *   xc = s                                                                     if last == NULL
 *   xc = c_last * last;  xc = fma(v[0], x0, xc);  xc = fma(v[k + 1], hist[k], xc) for k < n_hist   otherwise
 *   p  = c_xc * xc;  p = fma(u[0], x0, p);  p = fma(u[k + 1], hist[k], p) for k < min(n_hist, 2)
 *   prev_sample = p,  pred_x0 = x0,  corrected = xc.
 * hist is a host array of n_hist (0..B200_UNIPC_MAX_HIST) device pointers, the previous x0 estimates, newest first.
 * Any alignment; the outputs must not overlap the inputs or each other. */
int b200_unipc_step(const float* model_out, const float* sample, const float* last, const float* const* hist,
                    int32_t n_hist, const b200_unipc_coef* c, float* prev_sample, float* pred_x0, float* corrected,
                    int64_t n, void* stream);

/* SA-Solver's corrector and predictor for one step, each folded on the host in float64 and rounded once to fp32. */
typedef struct {
  float alpha_s, sigma_s;       /* of the current timestep, to form x0 as in b200_dpm_solver_step                */
  float c_last;                 /* corrector: weight of the previous step's start sample                         */
  float v[3];                   /* corrector: weights of x0 and of hist[0], hist[1]                              */
  float c_zlast;                /* corrector: weight of the previous step's noise                                */
  float c_xc;                   /* predictor: weight of the corrected sample                                     */
  float u[3];                   /* predictor: weights of x0 and of hist[0], hist[1]                              */
  float c_z;                    /* predictor: weight of this step's noise                                        */
  float clip_min, clip_max;
  int32_t prediction_type, clip;
} b200_sa_solver_coef;

/* b200_sa_solver_step: over n fp32 elements, with s = sample, m = model_out, in fp32:
 *   x0 as in b200_dpm_solver_step (prediction type, then the clip)
 *   xc = s                                                                     if last == NULL
 *   xc = c_last * last;  xc = fma(v[0], x0, xc);  xc = fma(v[k + 1], hist[k], xc) for k < n_hist;
 *        xc = fma(c_zlast, last_noise, xc) if last_noise != NULL                                      otherwise
 *   p  = c_xc * xc;  p = fma(u[0], x0, p);  p = fma(u[k + 1], hist[k], p) for k < n_hist;
 *        p = fma(c_z, noise, p) if noise != NULL
 *   prev_sample = p,  pred_x0 = x0,  corrected = xc.
 * hist is a host array of n_hist (0..B200_SA_SOLVER_MAX_HIST) device pointers, the previous x0 estimates, newest
 * first.  last_noise needs last.  Any alignment; the outputs must not overlap the inputs or each other. */
int b200_sa_solver_step(const float* model_out, const float* sample, const float* last, const float* last_noise,
                        const float* const* hist, int32_t n_hist, const float* noise, const b200_sa_solver_coef* c,
                        float* prev_sample, float* pred_x0, float* corrected, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GEN_SAMPLERS_H_ */
