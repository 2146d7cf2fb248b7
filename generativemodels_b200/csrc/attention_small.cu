// Small-shape attention on CUDA cores: softmax(scale * Q K^T) V with an online softmax, one warp per query row.
//
// Serves the shapes the tensor-core path is not built for: the test-suite head dims (2, 4, 8 ...), and
// cross-attention over a handful of context tokens (S = 1 in the classifier-free-guidance tutorial), where the
// whole problem is a few MFLOP.  Reference arithmetic: CrossAttention._attention
// (diffusion_model_unet.py:136-153) and AttentionBlock.forward (406-416): scores = scale * q.k, softmax over
// keys, probabilities times values.  Heads are channel slices [h*dh, (h+1)*dh) of the packed [B, T, H*dh] rows
// (reshape_heads_to_batch_dim, 107-116), so no head transpose is ever materialised.
#include "common.cuh"

namespace b200 {

template <int R>   // R = ceil(dh / 32) registers per lane
__global__ void attention_small_kernel(const h16* __restrict__ q, const h16* __restrict__ k,
                                       const h16* __restrict__ v, h16* __restrict__ out, int B,
                                       int T, int S, int heads, int dh, int q_pitch, int k_pitch, int v_pitch,
                                       int o_pitch, float scale, int kv_rows, int causal, int q_pos0,
                                       const int* __restrict__ pos_dev) {
  if (pos_dev) {                 // decode step captured in a CUDA graph: the prefix length lives in device memory
    q_pos0 = *pos_dev;
    S = q_pos0 + T;
  }
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total = (long long)B * heads * T;
  if (wid >= total) return;
  const int lane = threadIdx.x & 31;
  const int t = (int)(wid % T);
  const int h = (int)((wid / T) % heads);
  const int b = (int)(wid / ((long long)T * heads));
  const h16* qr = q + ((long long)b * T + t) * q_pitch + h * dh;
  float qreg[R], acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int d = lane + 32 * r;
    qreg[r] = d < dh ? h2f(qr[d]) * scale : 0.f;
    acc[r] = 0.f;
  }
  float mx = -INFINITY, denom = 0.f;
  // kv_rows = rows per batch item in the k / v buffers (a key/value cache holds max_seq rows, S of them valid);
  // causal: query t (absolute position q_pos0 + t) only sees keys s <= q_pos0 + t (SABlock causal_mask,
  // blocks/selfattention.py:93-97, 131-132)
  const h16* kb = k + (long long)b * kv_rows * k_pitch + h * dh;
  const h16* vb = v + (long long)b * kv_rows * v_pitch + h * dh;
  const int s_end = causal ? min(S, q_pos0 + t + 1) : S;
  for (int s = 0; s < s_end; ++s) {
    const h16* kr = kb + (long long)s * k_pitch;
    float dot = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int d = lane + 32 * r;
      if (d < dh) dot = fmaf(qreg[r], h2f(kr[d]), dot);
    }
    dot = warp_sum(dot);
    const float nmx = fmaxf(mx, dot);
    const float corr = __expf(mx - nmx);      // exp(-inf) = 0 on the first key
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
  const float inv = 1.0f / denom;
  h16* orow = out + ((long long)b * T + t) * o_pitch + h * dh;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int d = lane + 32 * r;
    if (d < dh) orow[d] = f2h(acc[r] * inv);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_attention_small(const void* q, const void* k, const void* v, void* out, int32_t B, int32_t T,
                                    int32_t S, int32_t heads, int32_t dh, int32_t q_pitch, int32_t k_pitch,
                                    int32_t v_pitch, int32_t o_pitch, float scale, void* stream_v) {
  return b200_attention_small_ex(q, k, v, out, B, T, S, heads, dh, q_pitch, k_pitch, v_pitch, o_pitch, scale, S, 0, 0,
                                 nullptr, stream_v);
}

extern "C" int b200_attention_small_ex(const void* q, const void* k, const void* v, void* out, int32_t B, int32_t T,
                                       int32_t S, int32_t heads, int32_t dh, int32_t q_pitch, int32_t k_pitch,
                                       int32_t v_pitch, int32_t o_pitch, float scale, int32_t kv_rows, int32_t causal,
                                       int32_t q_pos0, const int32_t* pos_dev, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(q && k && v && out && B >= 1 && T >= 1 && S >= 1 && heads >= 1 && dh >= 1, "attention_small: bad arguments");
  B200_CHECK_ARG((pos_dev || kv_rows >= S) && q_pos0 >= 0, "attention_small: kv_rows %d < S %d or negative query offset",
                 kv_rows, S);
  B200_CHECK_ARG(dh <= 1024, "attention_small: head_dim %d > 1024", dh);
  const long long total = (long long)B * heads * T;
  const int wpb = 8;
  const long long blocks = (total + wpb - 1) / wpb;
  B200_CHECK_ARG(blocks < (1ll << 31), "attention_small: too many rows");
  const h16* qq = reinterpret_cast<const h16*>(q);
  const h16* kk = reinterpret_cast<const h16*>(k);
  const h16* vv = reinterpret_cast<const h16*>(v);
  h16* oo = reinterpret_cast<h16*>(out);
#define LAUNCH(R) B200_CUDA(b200::launch_kernel(attention_small_kernel<R>, (unsigned)blocks, wpb * 32, 0, stream,  \
      qq, kk, vv, oo, B, T, S, heads, dh, q_pitch, k_pitch, v_pitch, o_pitch, scale, kv_rows, causal, q_pos0, pos_dev))
  if (dh <= 32) LAUNCH(1);
  else if (dh <= 64) LAUNCH(2);
  else if (dh <= 128) LAUNCH(4);
  else if (dh <= 256) LAUNCH(8);
  else if (dh <= 512) LAUNCH(16);
  else LAUNCH(32);
#undef LAUNCH
  B200_LAUNCH_CHECK("attention_small_kernel");
  return B200_OK;
}
