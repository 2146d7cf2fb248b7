// The multistep sampler steps.  DPM-Solver++ (DPMSolverMultistepScheduler.step): x0 from the model output, optional
// clip, then the update as one weighted sum of the sample, x0, up to two earlier x0 estimates and the noise.  UniPC
// (UniPCMultistepScheduler.step): the same x0, then the corrector as a weighted sum of the previous corrected sample, x0
// and up to three earlier x0 estimates, then the predictor from that.  SA-Solver (SASolverScheduler.step): the same x0,
// then the stochastic corrector from the previous step's start sample and noise, then the stochastic predictor from the
// corrected sample and this step's noise.  The host folds the solvers' formulas into those weights; the kernels only
// stream memory.  Contract: include/b200gen_samplers.h.
#include "common.cuh"
#include "../../include/b200gen_samplers.h"

namespace b200 {
namespace {

// x0 from the model output and the sample (every step kernel's first line): per prediction type, then the clip.
template <typename Coef>
__device__ __forceinline__ float form_x0(const Coef& c, float m, float s) {
  float x0;
  if (c.prediction_type == B200_PRED_EPSILON) x0 = fmaf(-c.sigma_s, m, s) / c.alpha_s;
  else if (c.prediction_type == B200_PRED_V) x0 = fmaf(c.alpha_s, s, -c.sigma_s * m);
  else x0 = m;
  if (c.clip) x0 = fminf(fmaxf(x0, c.clip_min), c.clip_max);
  return x0;
}

__device__ __forceinline__ void dpm_one(const b200_dpm_coef& c, float m, float s, float h0, float h1, float z, int nh,
                                        bool has_noise, float& p, float& x0) {
  x0 = form_x0(c, m, s);
  p = c.c_x * s;
  p = fmaf(c.w[0], x0, p);
  if (nh > 0) p = fmaf(c.w[1], h0, p);
  if (nh > 1) p = fmaf(c.w[2], h1, p);
  if (has_noise) p = fmaf(c.c_z, z, p);
}

__device__ __forceinline__ float4 ld4(const float* p, long long i) {
  return __ldg(reinterpret_cast<const float4*>(p) + i);
}

// Up to 7 fp32 streams per element: pure HBM streaming, so 128-bit accesses when every pointer is 16-byte aligned
// (VEC = 1) and a scalar tail for n % 4; VEC = 0 is the scalar path for any alignment.  NH = number of history tensors.
template <int VEC, int NH>
__global__ void __launch_bounds__(256) dpm_step_kernel(const float* __restrict__ m_in, const float* __restrict__ x,
                                                       const float* __restrict__ h0, const float* __restrict__ h1,
                                                       const float* __restrict__ noise, b200_dpm_coef c,
                                                       float* __restrict__ prev, float* __restrict__ x0_out,
                                                       long long n) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
  const bool has_noise = noise != nullptr;
  long long done = 0;
  if (VEC) {
    const long long nv = n >> 2;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i = tid; i < nv; i += nthr) {
      const float4 m = ld4(m_in, i), s = ld4(x, i);
      const float4 a = NH > 0 ? ld4(h0, i) : zero, b = NH > 1 ? ld4(h1, i) : zero;
      const float4 z = has_noise ? ld4(noise, i) : zero;
      float4 p, o;
      dpm_one(c, m.x, s.x, a.x, b.x, z.x, NH, has_noise, p.x, o.x);
      dpm_one(c, m.y, s.y, a.y, b.y, z.y, NH, has_noise, p.y, o.y);
      dpm_one(c, m.z, s.z, a.z, b.z, z.z, NH, has_noise, p.z, o.z);
      dpm_one(c, m.w, s.w, a.w, b.w, z.w, NH, has_noise, p.w, o.w);
      reinterpret_cast<float4*>(prev)[i] = p;
      reinterpret_cast<float4*>(x0_out)[i] = o;
    }
    done = nv << 2;
  }
  for (long long i = done + tid; i < n; i += nthr) {
    float p, o;
    dpm_one(c, m_in[i], x[i], NH > 0 ? h0[i] : 0.f, NH > 1 ? h1[i] : 0.f, has_noise ? noise[i] : 0.f, NH, has_noise,
            p, o);
    prev[i] = p;
    x0_out[i] = o;
  }
}

unsigned grid_for(long long work) {
  long long b = (work + 255) / 256;
  const long long cap = 16ll * sm_count();
  return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

template <int VEC>
cudaError_t launch(int nh, const float* m, const float* s, const float* h0, const float* h1, const float* z,
                   const b200_dpm_coef& c, float* prev, float* x0, long long n, cudaStream_t stream) {
  const unsigned grid = grid_for(VEC ? (n + 3) / 4 : n);
  if (nh == 0) return launch_kernel(dpm_step_kernel<VEC, 0>, grid, 256, 0, stream, m, s, h0, h1, z, c, prev, x0, n);
  if (nh == 1) return launch_kernel(dpm_step_kernel<VEC, 1>, grid, 256, 0, stream, m, s, h0, h1, z, c, prev, x0, n);
  return launch_kernel(dpm_step_kernel<VEC, 2>, grid, 256, 0, stream, m, s, h0, h1, z, c, prev, x0, n);
}

__device__ __forceinline__ void unipc_one(const b200_unipc_coef& c, float m, float s, float l, float h0, float h1,
                                          float h2, int nh, bool has_last, float& p, float& x0, float& xc) {
  x0 = form_x0(c, m, s);
  xc = s;
  if (has_last) {
    xc = c.c_last * l;
    xc = fmaf(c.v[0], x0, xc);
    if (nh > 0) xc = fmaf(c.v[1], h0, xc);
    if (nh > 1) xc = fmaf(c.v[2], h1, xc);
    if (nh > 2) xc = fmaf(c.v[3], h2, xc);
  }
  p = c.c_xc * xc;
  p = fmaf(c.u[0], x0, p);
  if (nh > 0) p = fmaf(c.u[1], h0, p);
  if (nh > 1) p = fmaf(c.u[2], h1, p);
}

// Up to 6 fp32 streams in and 3 out per element, vectorised as dpm_step_kernel.  NH = number of history tensors,
// LAST = whether the corrector runs (a previous corrected sample is given).
template <int VEC, int NH, bool LAST>
__global__ void __launch_bounds__(256) unipc_step_kernel(const float* __restrict__ m_in, const float* __restrict__ x,
                                                         const float* __restrict__ last, const float* __restrict__ h0,
                                                         const float* __restrict__ h1, const float* __restrict__ h2,
                                                         b200_unipc_coef c, float* __restrict__ prev,
                                                         float* __restrict__ x0_out, float* __restrict__ xc_out,
                                                         long long n) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
  long long done = 0;
  if (VEC) {
    const long long nv = n >> 2;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i = tid; i < nv; i += nthr) {
      const float4 m = ld4(m_in, i), s = ld4(x, i), l = LAST ? ld4(last, i) : zero;
      const float4 a = NH > 0 ? ld4(h0, i) : zero, b = NH > 1 ? ld4(h1, i) : zero, d = NH > 2 ? ld4(h2, i) : zero;
      float4 p, o, q;
      unipc_one(c, m.x, s.x, l.x, a.x, b.x, d.x, NH, LAST, p.x, o.x, q.x);
      unipc_one(c, m.y, s.y, l.y, a.y, b.y, d.y, NH, LAST, p.y, o.y, q.y);
      unipc_one(c, m.z, s.z, l.z, a.z, b.z, d.z, NH, LAST, p.z, o.z, q.z);
      unipc_one(c, m.w, s.w, l.w, a.w, b.w, d.w, NH, LAST, p.w, o.w, q.w);
      reinterpret_cast<float4*>(prev)[i] = p;
      reinterpret_cast<float4*>(x0_out)[i] = o;
      reinterpret_cast<float4*>(xc_out)[i] = q;
    }
    done = nv << 2;
  }
  for (long long i = done + tid; i < n; i += nthr) {
    float p, o, q;
    unipc_one(c, m_in[i], x[i], LAST ? last[i] : 0.f, NH > 0 ? h0[i] : 0.f, NH > 1 ? h1[i] : 0.f,
              NH > 2 ? h2[i] : 0.f, NH, LAST, p, o, q);
    prev[i] = p;
    x0_out[i] = o;
    xc_out[i] = q;
  }
}

template <int VEC, bool LAST>
cudaError_t launch_unipc_last(int nh, const float* m, const float* s, const float* l, const float* const* h,
                              const b200_unipc_coef& c, float* prev, float* x0, float* xc, long long n,
                              cudaStream_t stream) {
  const unsigned grid = grid_for(VEC ? (n + 3) / 4 : n);
  const float *h0 = h[0], *h1 = h[1], *h2 = h[2];
  if (nh == 0) return launch_kernel(unipc_step_kernel<VEC, 0, LAST>, grid, 256, 0, stream, m, s, l, h0, h1, h2, c, prev, x0, xc, n);
  if (nh == 1) return launch_kernel(unipc_step_kernel<VEC, 1, LAST>, grid, 256, 0, stream, m, s, l, h0, h1, h2, c, prev, x0, xc, n);
  if (nh == 2) return launch_kernel(unipc_step_kernel<VEC, 2, LAST>, grid, 256, 0, stream, m, s, l, h0, h1, h2, c, prev, x0, xc, n);
  return launch_kernel(unipc_step_kernel<VEC, 3, LAST>, grid, 256, 0, stream, m, s, l, h0, h1, h2, c, prev, x0, xc, n);
}

template <int VEC>
cudaError_t launch_unipc(int nh, const float* m, const float* s, const float* l, const float* const* h,
                         const b200_unipc_coef& c, float* prev, float* x0, float* xc, long long n, cudaStream_t stream) {
  if (l) return launch_unipc_last<VEC, true>(nh, m, s, l, h, c, prev, x0, xc, n, stream);
  return launch_unipc_last<VEC, false>(nh, m, s, l, h, c, prev, x0, xc, n, stream);
}

__device__ __forceinline__ void sa_one(const b200_sa_solver_coef& c, float m, float s, float l, float zl, float h0,
                                       float h1, float z, int nh, bool has_last, bool has_zl, bool has_z, float& p,
                                       float& x0, float& xc) {
  x0 = form_x0(c, m, s);
  xc = s;
  if (has_last) {
    xc = c.c_last * l;
    xc = fmaf(c.v[0], x0, xc);
    if (nh > 0) xc = fmaf(c.v[1], h0, xc);
    if (nh > 1) xc = fmaf(c.v[2], h1, xc);
    if (has_zl) xc = fmaf(c.c_zlast, zl, xc);
  }
  p = c.c_xc * xc;
  p = fmaf(c.u[0], x0, p);
  if (nh > 0) p = fmaf(c.u[1], h0, p);
  if (nh > 1) p = fmaf(c.u[2], h1, p);
  if (has_z) p = fmaf(c.c_z, z, p);
}

// Up to 7 fp32 streams in and 3 out per element, vectorised as dpm_step_kernel.  NH = number of history tensors,
// LAST = whether the corrector runs (the previous start sample is given); the two noise streams are optional.
template <int VEC, int NH, bool LAST>
__global__ void __launch_bounds__(256) sa_solver_step_kernel(const float* __restrict__ m_in,
                                                             const float* __restrict__ x,
                                                             const float* __restrict__ last,
                                                             const float* __restrict__ last_noise,
                                                             const float* __restrict__ h0,
                                                             const float* __restrict__ h1,
                                                             const float* __restrict__ noise, b200_sa_solver_coef c,
                                                             float* __restrict__ prev, float* __restrict__ x0_out,
                                                             float* __restrict__ xc_out, long long n) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
  const bool has_zl = LAST && last_noise != nullptr, has_z = noise != nullptr;
  long long done = 0;
  if (VEC) {
    const long long nv = n >> 2;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i = tid; i < nv; i += nthr) {
      const float4 m = ld4(m_in, i), s = ld4(x, i), l = LAST ? ld4(last, i) : zero;
      const float4 zl = has_zl ? ld4(last_noise, i) : zero, z = has_z ? ld4(noise, i) : zero;
      const float4 a = NH > 0 ? ld4(h0, i) : zero, b = NH > 1 ? ld4(h1, i) : zero;
      float4 p, o, q;
      sa_one(c, m.x, s.x, l.x, zl.x, a.x, b.x, z.x, NH, LAST, has_zl, has_z, p.x, o.x, q.x);
      sa_one(c, m.y, s.y, l.y, zl.y, a.y, b.y, z.y, NH, LAST, has_zl, has_z, p.y, o.y, q.y);
      sa_one(c, m.z, s.z, l.z, zl.z, a.z, b.z, z.z, NH, LAST, has_zl, has_z, p.z, o.z, q.z);
      sa_one(c, m.w, s.w, l.w, zl.w, a.w, b.w, z.w, NH, LAST, has_zl, has_z, p.w, o.w, q.w);
      reinterpret_cast<float4*>(prev)[i] = p;
      reinterpret_cast<float4*>(x0_out)[i] = o;
      reinterpret_cast<float4*>(xc_out)[i] = q;
    }
    done = nv << 2;
  }
  for (long long i = done + tid; i < n; i += nthr) {
    float p, o, q;
    sa_one(c, m_in[i], x[i], LAST ? last[i] : 0.f, has_zl ? last_noise[i] : 0.f, NH > 0 ? h0[i] : 0.f,
           NH > 1 ? h1[i] : 0.f, has_z ? noise[i] : 0.f, NH, LAST, has_zl, has_z, p, o, q);
    prev[i] = p;
    x0_out[i] = o;
    xc_out[i] = q;
  }
}

template <int VEC, bool LAST>
cudaError_t launch_sa_last(int nh, const float* m, const float* s, const float* l, const float* zl, const float* h0,
                           const float* h1, const float* z, const b200_sa_solver_coef& c, float* prev, float* x0,
                           float* xc, long long n, cudaStream_t stream) {
  const unsigned grid = grid_for(VEC ? (n + 3) / 4 : n);
  if (nh == 0) return launch_kernel(sa_solver_step_kernel<VEC, 0, LAST>, grid, 256, 0, stream, m, s, l, zl, h0, h1, z, c, prev, x0, xc, n);
  if (nh == 1) return launch_kernel(sa_solver_step_kernel<VEC, 1, LAST>, grid, 256, 0, stream, m, s, l, zl, h0, h1, z, c, prev, x0, xc, n);
  return launch_kernel(sa_solver_step_kernel<VEC, 2, LAST>, grid, 256, 0, stream, m, s, l, zl, h0, h1, z, c, prev, x0, xc, n);
}

template <int VEC>
cudaError_t launch_sa(int nh, const float* m, const float* s, const float* l, const float* zl, const float* h0,
                      const float* h1, const float* z, const b200_sa_solver_coef& c, float* prev, float* x0, float* xc,
                      long long n, cudaStream_t stream) {
  if (l) return launch_sa_last<VEC, true>(nh, m, s, l, zl, h0, h1, z, c, prev, x0, xc, n, stream);
  return launch_sa_last<VEC, false>(nh, m, s, l, zl, h0, h1, z, c, prev, x0, xc, n, stream);
}

}  // namespace
}  // namespace b200

extern "C" int b200_dpm_solver_step(const float* model_out, const float* sample, const float* const* hist,
                                    int32_t n_hist, const float* noise, const b200_dpm_coef* c, float* prev_sample,
                                    float* pred_x0, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(model_out && sample && c && prev_sample && pred_x0 && n >= 1, "dpm_solver_step: bad arguments");
  B200_CHECK_ARG(n_hist >= 0 && n_hist <= B200_DPM_MAX_HIST && (n_hist == 0 || hist),
                 "dpm_solver_step: n_hist must be 0..%d with a history array", B200_DPM_MAX_HIST);
  B200_CHECK_ARG(c->prediction_type == B200_PRED_EPSILON || c->prediction_type == B200_PRED_SAMPLE ||
                 c->prediction_type == B200_PRED_V, "dpm_solver_step: unknown prediction_type %d", c->prediction_type);
  const float* h[2] = {nullptr, nullptr};
  for (int k = 0; k < n_hist; ++k) {
    h[k] = hist[k];
    B200_CHECK_ARG(h[k], "dpm_solver_step: null history tensor %d", k);
  }
  const bool vec = (((uintptr_t)model_out | (uintptr_t)sample | (uintptr_t)h[0] | (uintptr_t)h[1] | (uintptr_t)noise |
                     (uintptr_t)prev_sample | (uintptr_t)pred_x0) & 15) == 0;
  if (vec) B200_CUDA(b200::launch<1>(n_hist, model_out, sample, h[0], h[1], noise, *c, prev_sample, pred_x0, n, stream));
  else B200_CUDA(b200::launch<0>(n_hist, model_out, sample, h[0], h[1], noise, *c, prev_sample, pred_x0, n, stream));
  B200_LAUNCH_CHECK("dpm_step_kernel");
  return B200_OK;
}

extern "C" int b200_unipc_step(const float* model_out, const float* sample, const float* last, const float* const* hist,
                               int32_t n_hist, const b200_unipc_coef* c, float* prev_sample, float* pred_x0,
                               float* corrected, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(model_out && sample && c && prev_sample && pred_x0 && corrected && n >= 1,
                 "unipc_step: bad arguments");
  B200_CHECK_ARG(n_hist >= 0 && n_hist <= B200_UNIPC_MAX_HIST && (n_hist == 0 || hist),
                 "unipc_step: n_hist must be 0..%d with a history array", B200_UNIPC_MAX_HIST);
  B200_CHECK_ARG(c->prediction_type == B200_PRED_EPSILON || c->prediction_type == B200_PRED_SAMPLE ||
                 c->prediction_type == B200_PRED_V, "unipc_step: unknown prediction_type %d", c->prediction_type);
  const float* h[3] = {nullptr, nullptr, nullptr};
  for (int k = 0; k < n_hist; ++k) {
    h[k] = hist[k];
    B200_CHECK_ARG(h[k], "unipc_step: null history tensor %d", k);
  }
  const bool vec = (((uintptr_t)model_out | (uintptr_t)sample | (uintptr_t)last | (uintptr_t)h[0] | (uintptr_t)h[1] |
                     (uintptr_t)h[2] | (uintptr_t)prev_sample | (uintptr_t)pred_x0 | (uintptr_t)corrected) & 15) == 0;
  if (vec) B200_CUDA(b200::launch_unipc<1>(n_hist, model_out, sample, last, h, *c, prev_sample, pred_x0, corrected, n,
                                           stream));
  else B200_CUDA(b200::launch_unipc<0>(n_hist, model_out, sample, last, h, *c, prev_sample, pred_x0, corrected, n,
                                       stream));
  B200_LAUNCH_CHECK("unipc_step_kernel");
  return B200_OK;
}

extern "C" int b200_sa_solver_step(const float* model_out, const float* sample, const float* last,
                                   const float* last_noise, const float* const* hist, int32_t n_hist,
                                   const float* noise, const b200_sa_solver_coef* c, float* prev_sample,
                                   float* pred_x0, float* corrected, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(model_out && sample && c && prev_sample && pred_x0 && corrected && n >= 1,
                 "sa_solver_step: bad arguments");
  B200_CHECK_ARG(last || !last_noise, "sa_solver_step: last_noise needs last");
  B200_CHECK_ARG(n_hist >= 0 && n_hist <= B200_SA_SOLVER_MAX_HIST && (n_hist == 0 || hist),
                 "sa_solver_step: n_hist must be 0..%d with a history array", B200_SA_SOLVER_MAX_HIST);
  B200_CHECK_ARG(c->prediction_type == B200_PRED_EPSILON || c->prediction_type == B200_PRED_SAMPLE ||
                 c->prediction_type == B200_PRED_V, "sa_solver_step: unknown prediction_type %d", c->prediction_type);
  const float* h[2] = {nullptr, nullptr};
  for (int k = 0; k < n_hist; ++k) {
    h[k] = hist[k];
    B200_CHECK_ARG(h[k], "sa_solver_step: null history tensor %d", k);
  }
  const bool vec = (((uintptr_t)model_out | (uintptr_t)sample | (uintptr_t)last | (uintptr_t)last_noise |
                     (uintptr_t)h[0] | (uintptr_t)h[1] | (uintptr_t)noise | (uintptr_t)prev_sample |
                     (uintptr_t)pred_x0 | (uintptr_t)corrected) & 15) == 0;
  if (vec) B200_CUDA(b200::launch_sa<1>(n_hist, model_out, sample, last, last_noise, h[0], h[1], noise, *c,
                                        prev_sample, pred_x0, corrected, n, stream));
  else B200_CUDA(b200::launch_sa<0>(n_hist, model_out, sample, last, last_noise, h[0], h[1], noise, *c, prev_sample,
                                    pred_x0, corrected, n, stream));
  B200_LAUNCH_CHECK("sa_solver_step_kernel");
  return B200_OK;
}
