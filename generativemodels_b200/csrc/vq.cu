// VectorQuantizer nearest-codebook search (vector_quantizer.py:86-138, 183-186, 212-218).
//
// The reference materialises an M x K distance matrix (torch.mm + broadcasts), takes torch.max(-d) and builds an
// M x K one-hot.  Here: the codebook (and |e|^2) sits in shared memory, one warp owns one input vector at a time,
// every lane scans K/32 codes with fp32 FMAs in a fixed order, and a warp-shuffle (distance, index) argmin picks
// the winner — ties go to the lowest index exactly like torch.max.  The winner's row is gathered straight away
// (bf16 for the decoder, fp32 with the straight-through rounding for the API), the commitment-loss numerator and
// the code histogram (perplexity) are accumulated on the way.  HBM traffic = M*D*4 read + M*8 (+ M*D*{2,4}) write.
#include "common.cuh"
#include <mutex>

namespace b200 {

static constexpr int kVqWarps = 8;

__global__ void vq_argmin_kernel(const float* __restrict__ x, long long M, int D, int x_pitch,
                                 const float* __restrict__ cb, int K, long long* __restrict__ idx_out,
                                 h16* __restrict__ q16, int q_pitch, float* __restrict__ q32, int ste,
                                 double* __restrict__ sqerr, int* __restrict__ hist) {
  extern __shared__ float sm[];
  const int DP = D + 1;                       // padded pitch: lanes hit distinct banks
  float* s_cb = sm;                           // [K][DP]
  float* s_ee = s_cb + (size_t)K * DP;        // [K]
  float* s_x = s_ee + K;                      // [warps][D]
  for (int i = threadIdx.x; i < K * D; i += blockDim.x) s_cb[(i / D) * DP + i % D] = cb[i];
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    // (embedding.weight.t() ** 2).sum(dim=0): sequential over the embedding dimension
    float e = 0.f;
    for (int d = 0; d < D; ++d) e += s_cb[k * DP + d] * s_cb[k * DP + d];
    s_ee[k] = e;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* xs = s_x + warp * D;
  double err_acc = 0.0;
  for (long long m = (long long)blockIdx.x * kVqWarps + warp; m < M; m += (long long)gridDim.x * kVqWarps) {
    const float* xr = x + m * x_pitch;
    float xx = 0.f;
    for (int d = lane; d < D; d += 32) {
      const float v = xr[d];
      xs[d] = v;
    }
    __syncwarp();
    for (int d = 0; d < D; ++d) xx += xs[d] * xs[d];     // every lane: same sequential |x|^2
    float best = INFINITY;
    int bi = 0x7fffffff;
    for (int k = lane; k < K; k += 32) {
      const float* e = s_cb + k * DP;
      float dot = 0.f;
      for (int d = 0; d < D; ++d) dot = fmaf(xs[d], e[d], dot);
      const float dist = (xx + s_ee[k]) - 2.0f * dot;
      if (dist < best) { best = dist; bi = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (bi == 0x7fffffff) bi = 0;   // all-NaN row
    if (lane == 0) {
      idx_out[m] = bi;
      if (hist) atomicAdd(hist + bi, 1);
    }
    const float* e = s_cb + bi * DP;
    for (int d = lane; d < D; d += 32) {
      const float qv = e[d], xv = xs[d];
      if (q16) q16[m * q_pitch + d] = f2h(qv);
      if (q32) q32[m * D + d] = ste ? xv + (qv - xv) : qv;
      if (sqerr) { const float df = qv - xv; err_acc += (double)df * (double)df; }
    }
    if (q16)
      for (int d = D + lane; d < q_pitch; d += 32) q16[m * q_pitch + d] = f2h(0.f);
    __syncwarp();
  }
  if (sqerr) {
    for (int o = 16; o > 0; o >>= 1) err_acc += __shfl_xor_sync(0xffffffffu, err_acc, o);
    if (lane == 0 && err_acc != 0.0) atomicAdd(sqerr, err_acc);
  }
}

// Register-tiled variant for embedding_dim == DD (32: the VQ-VAE tutorial's codebook): the generic kernel above issues
// two shared-memory loads per FMA (x[d] broadcast + e[d]) and is bound by the shared-memory port at ~1/8 of the fp32
// rate.  Here a warp owns RR input vectors at a time and every lane keeps all
// RR x DD of their components in registers, so each e[d] load feeds RR FMAs.  Arithmetic per (vector, code) is the
// same fixed-order fp32 sequence as the generic kernel — indices are bit-identical.
template <int DD, int RR>
__global__ void __launch_bounds__(kVqWarps * 32) vq_argmin_tiled_kernel(
    const float* __restrict__ x, long long M, int x_pitch, const float* __restrict__ cb, int K,
    long long* __restrict__ idx_out, h16* __restrict__ q16, int q_pitch, float* __restrict__ q32, int ste,
    double* __restrict__ sqerr, int* __restrict__ hist) {
  extern __shared__ float sm[];
  constexpr int DP = DD + 1;
  float* s_cb = sm;                           // [K][DP]
  float* s_ee = s_cb + (size_t)K * DP;        // [K]
  for (int i = threadIdx.x; i < K * DD; i += blockDim.x) s_cb[(i / DD) * DP + i % DD] = cb[i];
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float e = 0.f;
    for (int d = 0; d < DD; ++d) e += s_cb[k * DP + d] * s_cb[k * DP + d];
    s_ee[k] = e;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double err_acc = 0.0;
  const long long groups = (M + RR - 1) / RR;
  for (long long g = (long long)blockIdx.x * kVqWarps + warp; g < groups; g += (long long)gridDim.x * kVqWarps) {
    float xv[RR][DD], xx[RR], best[RR];
    int bi[RR];
#pragma unroll
    for (int r = 0; r < RR; ++r) {
      long long m = g * RR + r;
      if (m >= M) m = M - 1;                  // duplicate of the last vector: computed, never written
      const float* xr = x + m * x_pitch;
#pragma unroll
      for (int d = 0; d < DD; ++d) xv[r][d] = __ldg(xr + d);      // same address in every lane: one broadcast request
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < DD; ++d) acc += xv[r][d] * xv[r][d];
      xx[r] = acc;
      best[r] = INFINITY;
      bi[r] = 0x7fffffff;
    }
    for (int k = lane; k < K; k += 32) {
      const float* e = s_cb + k * DP;
      float dot[RR];
#pragma unroll
      for (int r = 0; r < RR; ++r) dot[r] = 0.f;
#pragma unroll
      for (int d = 0; d < DD; ++d) {
        const float ev = e[d];
#pragma unroll
        for (int r = 0; r < RR; ++r) dot[r] = fmaf(xv[r][d], ev, dot[r]);
      }
      const float ee = s_ee[k];
#pragma unroll
      for (int r = 0; r < RR; ++r) {
        const float dist = (xx[r] + ee) - 2.0f * dot[r];
        if (dist < best[r]) { best[r] = dist; bi[r] = k; }
      }
    }
#pragma unroll
    for (int r = 0; r < RR; ++r) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best[r], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[r], o);
        if (ob < best[r] || (ob == best[r] && oi < bi[r])) { best[r] = ob; bi[r] = oi; }
      }
      if (bi[r] == 0x7fffffff) bi[r] = 0;     // all-NaN row
      const long long m = g * RR + r;
      if (m < M) {
        if (lane == 0) {
          idx_out[m] = bi[r];
          if (hist) atomicAdd(hist + bi[r], 1);
        }
        const float* e = s_cb + bi[r] * DP;
        for (int d = lane; d < DD; d += 32) {
          const float qv = e[d];
          float xd = 0.f;
#pragma unroll
          for (int t = 0; t < DD; ++t) if (t == d) xd = xv[r][t];          // register file has no dynamic index
          if (q16) q16[m * q_pitch + d] = f2h(qv);
          if (q32) q32[m * DD + d] = ste ? xd + (qv - xd) : qv;
          if (sqerr) { const float df = qv - xd; err_acc += (double)df * (double)df; }
        }
        if (q16)
          for (int d = DD + lane; d < q_pitch; d += 32) q16[m * q_pitch + d] = f2h(0.f);
      }
    }
  }
  if (sqerr) {
    for (int o = 16; o > 0; o >>= 1) err_acc += __shfl_xor_sync(0xffffffffu, err_acc, o);
    if (lane == 0 && err_acc != 0.0) atomicAdd(sqerr, err_acc);
  }
}

__global__ void vq_gather_kernel(const long long* __restrict__ idx, long long M, const float* __restrict__ cb, int K,
                                 int D, h16* __restrict__ q16, int q_pitch) {
  const long long total = M * q_pitch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / q_pitch;
    const int d = (int)(i % q_pitch);
    long long k = idx[m];
    if (k < 0) k = 0;
    if (k >= K) k = K - 1;
    q16[i] = f2h(d < D ? cb[k * D + d] : 0.f);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_vq_argmin_gather(const float* x, int64_t M, int32_t D, int32_t x_pitch, const float* codebook,
                                     int32_t K, int64_t* indices, void* q_h16, int32_t q_pitch, float* q_f32,
                                     int32_t ste, double* sqerr_sum, int32_t* hist, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && codebook && indices && M >= 1 && D >= 1 && K >= 1 && x_pitch >= D, "vq_argmin: bad arguments");
  B200_CHECK_ARG(!q_h16 || q_pitch >= D, "vq_argmin: q_pitch %d < D %d", q_pitch, D);
  const size_t smem = ((size_t)K * (D + 1) + K + (size_t)kVqWarps * D) * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("vq_argmin: codebook %d x %d does not fit in shared memory", K, D);
    return B200_ENOTSUP;
  }
  // once, to the largest codebook accepted above (read-only afterwards: the entry point stays re-entrant)
  static std::once_flag attr_once;
  static cudaError_t attr_rc = cudaSuccess;
  std::call_once(attr_once, [] {
    attr_rc = cudaFuncSetAttribute(vq_argmin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (attr_rc == cudaSuccess)
      attr_rc = cudaFuncSetAttribute(vq_argmin_tiled_kernel<32, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  });
  B200_CUDA(attr_rc);
  if (D == 32) {
    // register-tiled path: 4 vectors per warp iteration
    long long blocks = ((M + 3) / 4 + kVqWarps - 1) / kVqWarps;
    const long long cap = 2ll * sm_count();
    if (blocks > cap) blocks = cap;
    const size_t smem_t = ((size_t)K * (D + 1) + K) * sizeof(float);
    B200_CUDA(b200::launch_kernel(vq_argmin_tiled_kernel<32, 4>, (unsigned)blocks, kVqWarps * 32, smem_t, stream, x, (long long)M, x_pitch,
                               codebook, K, reinterpret_cast<long long*>(indices), reinterpret_cast<h16*>(q_h16), q_pitch,
                               q_f32, ste, sqerr_sum, hist));
    B200_LAUNCH_CHECK("vq_argmin_tiled_kernel");
    return B200_OK;
  }
  long long blocks = (M + kVqWarps - 1) / kVqWarps;
  const long long cap = 2ll * sm_count();
  if (blocks > cap) blocks = cap;
  B200_CUDA(b200::launch_kernel(vq_argmin_kernel, (unsigned)blocks, kVqWarps * 32, smem, stream,
      x, (long long)M, D, x_pitch, codebook, K, reinterpret_cast<long long*>(indices), reinterpret_cast<h16*>(q_h16),
      q_pitch, q_f32, ste, sqerr_sum, hist));
  B200_LAUNCH_CHECK("vq_argmin_kernel");
  return B200_OK;
}

extern "C" int b200_vq_gather(const int64_t* indices, int64_t M, const float* codebook, int32_t K, int32_t D,
                              void* q_h16, int32_t q_pitch, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(indices && codebook && q_h16 && M >= 1 && q_pitch >= D, "vq_gather: bad arguments");
  long long blocks = (M * q_pitch + 255) / 256;
  const long long cap = 8ll * sm_count();
  if (blocks > cap) blocks = cap;
  B200_CUDA(b200::launch_kernel(vq_gather_kernel, (unsigned)blocks, 256, 0, stream, reinterpret_cast<const long long*>(indices), M, codebook, K, D,
                                                         reinterpret_cast<h16*>(q_h16), q_pitch));
  B200_LAUNCH_CHECK("vq_gather_kernel");
  return B200_OK;
}
