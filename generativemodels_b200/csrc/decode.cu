// Batch-of-a-few-rows kernels for autoregressive decoding (VQVAETransformerInferer.sample, inferer.py:1183-1245).
//
// One new token per sequence means every linear layer is a GEMV: 2 * K * O FLOPs against K * O * 2 bytes of weights,
// i.e. HBM/L2-bound by a factor of ~1000 — the 128-row tensor-core tile of b200_igemm spends its pipeline latency
// on 0.5 MFLOP.  These kernels read each weight row once with 16-byte loads, keep the (optionally LayerNorm-ed)
// activation rows in shared memory and finish with the same fused epilogue (bias, GELU, residual), so a decode step
// is ~100 launches of a few microseconds that replay from one CUDA graph.
#include "common.cuh"

namespace b200 {

static constexpr int kRowsMax = 8;

// y[m, o] = act( LN?(x[m, :]) . W[o, :] + bias[o] ) + res[m, o]      (m < M <= 8; W bf16 K-major, row pitch w_pitch)
__global__ void __launch_bounds__(256) rows_linear_kernel(const h16* __restrict__ x, int x_pitch, int M, int K,
                                                          const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                                                          float ln_eps, const h16* __restrict__ W, int w_pitch,
                                                          int O, const float* __restrict__ bias, int act,
                                                          const h16* __restrict__ res, int r_pitch, void* out,
                                                          int o_pitch, int out_f32) {
  extern __shared__ __align__(16) uint8_t dsm[];
  h16* xs = reinterpret_cast<h16*>(dsm);        // [M][Kp], Kp = K rounded up to 8
  const int Kp = (K + 7) & ~7;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // ---- stage the rows (LayerNorm applied on the way in, rounded to bf16 like the stand-alone kernel's output) ----
  for (int m = warp; m < M; m += 8) {
    const h16* xr = x + (long long)m * x_pitch;
    if (ln_g) {
      // two passes, as layernorm_kernel: the variance from x - mean, not E[x^2] - mean^2 (which cancels when the
      // row's mean is large against its spread)
      float s = 0.f;
      for (int k = lane; k < K; k += 32) s += h2f(xr[k]);
      const float mean = warp_sum(s) / K;
      float q = 0.f;
      for (int k = lane; k < K; k += 32) {
        const float d = h2f(xr[k]) - mean;
        q = fmaf(d, d, q);
      }
      const float rstd = rsqrtf(warp_sum(q) / K + ln_eps);
      for (int k = lane; k < Kp; k += 32)
        xs[m * Kp + k] = k < K ? f2h((h2f(xr[k]) - mean) * rstd * ln_g[k] + ln_b[k])
                               : f2h(0.f);
    } else {
      for (int k = lane; k < Kp; k += 32) xs[m * Kp + k] = k < K ? xr[k] : f2h(0.f);
    }
  }
  __syncthreads();
  // ---- one output column per warp per pass ----
  for (int o = blockIdx.x * 8 + warp; o < O; o += gridDim.x * 8) {
    const h16* wr = W + (long long)o * w_pitch;
    float acc[kRowsMax];
#pragma unroll
    for (int m = 0; m < kRowsMax; ++m) acc[m] = 0.f;
    for (int k0 = lane * 8; k0 < Kp; k0 += 256) {
      float wf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(wr + k0)), wf);
#pragma unroll
      for (int m = 0; m < kRowsMax; ++m) {
        if (m < M) {
          float xf[8];
          unpack8(*reinterpret_cast<const uint4*>(xs + m * Kp + k0), xf);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[m] = fmaf(xf[e], wf[e], acc[m]);
        }
      }
    }
#pragma unroll
    for (int m = 0; m < kRowsMax; ++m)
      if (m < M) acc[m] = warp_sum(acc[m]);
    if (lane < M) {
      float v = 0.f;
#pragma unroll
      for (int m = 0; m < kRowsMax; ++m)
        if (m == lane) v = acc[m];
      if (bias) v += bias[o];
      v = apply_act(v, act);
      if (res) v += h2f(res[(long long)lane * r_pitch + o]);
      if (out_f32) reinterpret_cast<float*>(out)[(long long)lane * o_pitch + o] = v;
      else reinterpret_cast<h16*>(out)[(long long)lane * o_pitch + o] = f2h(v);
    }
  }
}

// One query row per (batch, head) over S cached keys: 8 warps split the keys, each keeps an online-softmax state,
// the states are merged through shared memory.  S (and the causal horizon) may come from device memory.
template <int R>
__global__ void __launch_bounds__(256) attention_decode_kernel(const h16* __restrict__ q,
                                                               const h16* __restrict__ k,
                                                               const h16* __restrict__ v,
                                                               h16* __restrict__ out, int S, int heads, int dh,
                                                               int q_pitch, int k_pitch, int v_pitch, int o_pitch,
                                                               float scale, int kv_rows, const int* __restrict__ pos_dev) {
  if (pos_dev) S = *pos_dev + 1;
  const int h = blockIdx.x % heads, b = blockIdx.x / heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const h16* qr = q + (long long)b * q_pitch + h * dh;
  float qreg[R], acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int d = lane + 32 * r;
    qreg[r] = d < dh ? h2f(qr[d]) * scale : 0.f;
    acc[r] = 0.f;
  }
  float mx = -INFINITY, denom = 0.f;
  const h16* kb = k + (long long)b * kv_rows * k_pitch + h * dh;
  const h16* vb = v + (long long)b * kv_rows * v_pitch + h * dh;
  for (int s = warp; s < S; s += 8) {
    const h16* kr = kb + (long long)s * k_pitch;
    float dot = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int d = lane + 32 * r;
      if (d < dh) dot = fmaf(qreg[r], h2f(kr[d]), dot);
    }
    dot = warp_sum(dot);
    const float nmx = fmaxf(mx, dot);
    const float corr = __expf(mx - nmx);
    const float p = __expf(dot - nmx);
    denom = denom * corr + p;
    const h16* vr = vb + (long long)s * v_pitch;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int d = lane + 32 * r;
      if (d < dh) acc[r] = acc[r] * corr + p * h2f(vr[d]);
    }
    mx = nmx;
  }
  __shared__ float s_mx[8], s_den[8];
  __shared__ float s_acc[8][32 * R];
  if (lane == 0) { s_mx[warp] = mx; s_den[warp] = denom; }
#pragma unroll
  for (int r = 0; r < R; ++r) s_acc[warp][lane + 32 * r] = acc[r];
  __syncthreads();
  if (warp == 0) {
    float gm = -INFINITY;
#pragma unroll
    for (int w = 0; w < 8; ++w) gm = fmaxf(gm, s_mx[w]);
    float den = 0.f;
    float o[R];
#pragma unroll
    for (int r = 0; r < R; ++r) o[r] = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const float c = s_mx[w] == -INFINITY ? 0.f : __expf(s_mx[w] - gm);
      den += s_den[w] * c;
#pragma unroll
      for (int r = 0; r < R; ++r) o[r] += s_acc[w][lane + 32 * r] * c;
    }
    const float inv = 1.0f / den;
    h16* orow = out + (long long)b * o_pitch + h * dh;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int d = lane + 32 * r;
      if (d < dh) orow[d] = f2h(o[r] * inv);
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_rows_linear(const void* x, int32_t x_pitch, int32_t M, int32_t K, const float* ln_gamma,
                                const float* ln_beta, float ln_eps, const void* w, int32_t w_pitch, int32_t O,
                                const float* bias, int32_t act, const void* res, int32_t r_pitch, void* out,
                                int32_t o_pitch, int32_t out_dtype, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && w && out && M >= 1 && M <= kRowsMax && K >= 1 && O >= 1, "rows_linear: 1 <= M <= 8 rows");
  B200_CHECK_ARG(w_pitch % 8 == 0 && w_pitch >= ((K + 7) & ~7) && ((uintptr_t)w % 16) == 0 && x_pitch >= K &&
                 o_pitch >= O && (!res || r_pitch >= O) && (!ln_gamma || ln_beta),
                 "rows_linear: weights must be 16-byte aligned K-major rows with pitch >= K (multiple of 8)");
  const int smem = M * ((K + 7) & ~7) * 2;
  B200_CHECK_ARG(smem <= 48 * 1024, "rows_linear: M * K too large (%d bytes of rows)", smem);
  int blocks = (O + 7) / 8;
  if (blocks > 8 * sm_count()) blocks = 8 * sm_count();
  B200_CUDA(b200::launch_kernel(rows_linear_kernel, blocks, 256, smem, stream, 
      reinterpret_cast<const h16*>(x), x_pitch, M, K, ln_gamma, ln_beta, ln_eps,
      reinterpret_cast<const h16*>(w), w_pitch, O, bias, act, reinterpret_cast<const h16*>(res),
      r_pitch, out, o_pitch, out_dtype == B200_DT_F32 ? 1 : 0));
  B200_LAUNCH_CHECK("rows_linear_kernel");
  return B200_OK;
}

extern "C" int b200_attention_decode(const void* q, const void* k, const void* v, void* out, int32_t B, int32_t S,
                                     int32_t heads, int32_t dh, int32_t q_pitch, int32_t k_pitch, int32_t v_pitch,
                                     int32_t o_pitch, float scale, int32_t kv_rows, const int32_t* pos_dev,
                                     void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(q && k && v && out && B >= 1 && heads >= 1 && dh >= 1 && dh <= 256 && (pos_dev || (S >= 1 && S <= kv_rows)),
                 "attention_decode: bad arguments (head_dim <= 256)");
  const h16* qq = reinterpret_cast<const h16*>(q);
  const h16* kk = reinterpret_cast<const h16*>(k);
  const h16* vv = reinterpret_cast<const h16*>(v);
  h16* oo = reinterpret_cast<h16*>(out);
#define LAUNCH(R) B200_CUDA(b200::launch_kernel(attention_decode_kernel<R>, B * heads, 256, 0, stream, qq, kk, vv, oo, S, heads, dh, q_pitch, k_pitch, \
                                                                          v_pitch, o_pitch, scale, kv_rows, pos_dev))
  if (dh <= 32) LAUNCH(1);
  else if (dh <= 64) LAUNCH(2);
  else if (dh <= 128) LAUNCH(4);
  else LAUNCH(8);
#undef LAUNCH
  B200_LAUNCH_CHECK("attention_decode_kernel");
  return B200_OK;
}
