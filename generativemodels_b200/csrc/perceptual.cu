// Perceptual distance (generative/losses/perceptual.py of the reference, network_type="resnet50"): the input
// preparation in front of the ResNet-50 feature network (1 -> 3 channel repeat, ImageNet z-score, the 2.5-D slice
// gather) and the channel-normalised feature distance behind it.  Contracts: include/b200gen_perceptual.h.
#include "common.cuh"
#include "../../include/b200gen_perceptual.h"

namespace b200 {
namespace {

constexpr int kThreads = 256;

struct PrepSide {
  const void* x;
  int dt;
  long long st[5];
  uint4* out;
};

// One thread per output pixel of one input (blockIdx.y): three z-scored channels and five zero channels, one 16-byte
// store.
__global__ void __launch_bounds__(kThreads) perceptual_prep_kernel(PrepSide a, PrepSide b, int C, int S, int OH,
                                                                    int OW, const int64_t* __restrict__ idx,
                                                                    long long total) {
  const bool first = blockIdx.y == 0;
  const void* src = first ? a.x : b.x;
  const int dt = first ? a.dt : b.dt;
  long long st[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) st[k] = first ? a.st[k] : b.st[k];
  uint4* out = first ? a.out : b.out;
  const float mean[3] = {0.485f, 0.456f, 0.406f};
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long img = i / ((long long)OH * OW);
    const int r = (int)(i - img * OH * OW);
    const int h = r / OW, w = r - h * OW;
    const long long q = idx ? idx[img] : img;
    const long long base = (q / S) * st[0] + (q % S) * st[2] + h * st[3] + w * st[4];
    float v[8];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = load_any(src, dt, base + (C == 1 ? 0 : c) * st[1]);
      v[c] = __fdiv_rn(__fsub_rn(x, mean[c]), stdv[c]);
    }
#pragma unroll
    for (int c = 3; c < 8; ++c) v[c] = 0.f;
    out[i] = pack8(v);
  }
}

template <int DT>
__device__ __forceinline__ float feat(const void* p, long long i) {
  if (DT == B200_DT_F32) return static_cast<const float*>(p)[i];
  return h2f(static_cast<const h16*>(p)[i]);
}

// Butterfly sum: every lane ends with the same bits (each level adds the same two values on both partners).
__device__ __forceinline__ float lane_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per pixel: the two norms, then the squared difference of the normalised vectors.
template <int DT>
__global__ void __launch_bounds__(kThreads) perceptual_pixel_kernel(const void* __restrict__ x,
                                                                     const void* __restrict__ y, long long rows, int C,
                                                                     int pitch, float* __restrict__ pixel) {
  const int lane = threadIdx.x % 32;
  const long long row = (long long)blockIdx.x * (kThreads / 32) + threadIdx.x / 32;
  if (row >= rows) return;
  const long long base = row * pitch;
  float sx = 0.f, sy = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float a = feat<DT>(x, base + c), b = feat<DT>(y, base + c);
    sx = __fmaf_rn(a, a, sx);
    sy = __fmaf_rn(b, b, sy);
  }
  const float ix = __fadd_rn(__fsqrt_rn(lane_sum(sx)), B200_PERCEPTUAL_EPS);
  const float iy = __fadd_rn(__fsqrt_rn(lane_sum(sy)), B200_PERCEPTUAL_EPS);
  float sd = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = __fsub_rn(__fdiv_rn(feat<DT>(x, base + c), ix), __fdiv_rn(feat<DT>(y, base + c), iy));
    sd = __fmaf_rn(d, d, sd);
  }
  sd = lane_sum(sd);
  if (lane == 0) pixel[row] = sd;
}

// One block per image: fp64 sum of its pixels (thread t takes p = t, t + 256, ... in order; then the warps'
// butterflies and warp 0's fixed-order sum of the eight warp sums), divided by HW.
__global__ void __launch_bounds__(kThreads) perceptual_image_kernel(const float* __restrict__ pixel, int HW,
                                                                     double* __restrict__ image,
                                                                     float* __restrict__ image32) {
  __shared__ double red[kThreads / 32];
  const float* p = pixel + (long long)blockIdx.x * HW;
  double s = 0.0;
  for (int i = threadIdx.x; i < HW; i += kThreads) s += (double)p[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    const double m = t / (double)HW;
    image[blockIdx.x] = m;
    if (image32) image32[blockIdx.x] = (float)m;
  }
}

struct Counts {
  int n[3];
};

__global__ void perceptual_mean_kernel(const double* __restrict__ image, int n_groups, Counts c, double* means,
                                       float* loss) {
  double total = 0.0;
  const double* g = image;
  for (int k = 0; k < n_groups; ++k) {
    double s = 0.0;
    for (int i = 0; i < c.n[k]; ++i) s += g[i];
    const double m = s / (double)c.n[k];
    means[k] = m;
    total += m;
    g += c.n[k];
  }
  means[n_groups] = total;
  *loss = (float)total;
}

bool input_dtype_ok(int dt) {
  return dt == B200_DT_F32 || dt == B200_DT_F64 || dt == B200_DT_FP16 || dt == B200_DT_BF16;
}

}  // namespace
}  // namespace b200

extern "C" int b200_perceptual_prep(const void* x, int32_t x_dtype, const int64_t* x_strides, const void* y,
                                    int32_t y_dtype, const int64_t* y_strides, int32_t C, int32_t S, int32_t OH,
                                    int32_t OW, const int64_t* idx, int32_t n_out, void* out_x, void* out_y,
                                    void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && x_strides && y_strides && out_x && out_y, "perceptual_prep: null pointer");
  B200_CHECK_ARG(b200::input_dtype_ok(x_dtype) && b200::input_dtype_ok(y_dtype),
                 "perceptual_prep: unknown dtype %d / %d", x_dtype, y_dtype);
  B200_CHECK_ARG(C == 1 || C == 3, "perceptual_prep: C must be 1 or 3, got %d", C);
  B200_CHECK_ARG(S >= 1 && OH >= 1 && OW >= 1 && n_out >= 1, "perceptual_prep: bad extents");
  B200_CHECK_ARG(((uintptr_t)out_x % 16) == 0 && ((uintptr_t)out_y % 16) == 0, "perceptual_prep: unaligned output");
  b200::PrepSide a{x, x_dtype, {}, static_cast<uint4*>(out_x)}, b{y, y_dtype, {}, static_cast<uint4*>(out_y)};
  for (int i = 0; i < 5; ++i) {
    a.st[i] = x_strides[i];
    b.st[i] = y_strides[i];
  }
  const long long total = (long long)n_out * OH * OW;
  long long blocks = (total + b200::kThreads - 1) / b200::kThreads;
  const long long cap = 16ll * b200::sm_count();
  if (blocks > cap) blocks = cap;
  B200_CUDA(b200::launch_kernel(b200::perceptual_prep_kernel, dim3((unsigned)blocks, 2), dim3(b200::kThreads), 0,
                                stream, a, b, (int)C, (int)S, (int)OH, (int)OW, idx, total));
  B200_LAUNCH_CHECK("perceptual_prep_kernel");
  return B200_OK;
}

extern "C" int b200_perceptual_distance(const void* x, const void* y, int32_t dtype, int32_t B, int32_t HW, int32_t C,
                                        int32_t pitch, float* pixel, double* image, float* image32, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && pixel && image, "perceptual_distance: null pointer");
  B200_CHECK_ARG(dtype == B200_DT_F32 || dtype == B200_DT_H16, "perceptual_distance: dtype must be F32 or H16");
  B200_CHECK_ARG(B >= 1 && HW >= 1 && C >= 1 && pitch >= C, "perceptual_distance: bad extents");
  const long long rows = (long long)B * HW;
  const long long blocks = (rows + b200::kThreads / 32 - 1) / (b200::kThreads / 32);
  B200_CHECK_ARG(blocks < (1ll << 31), "perceptual_distance: too many pixels");
  if (dtype == B200_DT_F32)
    B200_CUDA(b200::launch_kernel(b200::perceptual_pixel_kernel<B200_DT_F32>, dim3((unsigned)blocks),
                                  dim3(b200::kThreads), 0, stream, x, y, rows, (int)C, (int)pitch, pixel));
  else
    B200_CUDA(b200::launch_kernel(b200::perceptual_pixel_kernel<B200_DT_H16>, dim3((unsigned)blocks),
                                  dim3(b200::kThreads), 0, stream, x, y, rows, (int)C, (int)pitch, pixel));
  B200_LAUNCH_CHECK("perceptual_pixel_kernel");
  B200_CUDA(b200::launch_kernel(b200::perceptual_image_kernel, dim3(B), dim3(b200::kThreads), 0, stream,
                                (const float*)pixel, (int)HW, image, image32));
  B200_LAUNCH_CHECK("perceptual_image_kernel");
  return B200_OK;
}

extern "C" int b200_perceptual_mean(const double* image, int32_t n_groups, const int32_t* counts, double* means,
                                    float* loss, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(image && counts && means && loss, "perceptual_mean: null pointer");
  B200_CHECK_ARG(n_groups >= 1 && n_groups <= 3, "perceptual_mean: 1 to 3 groups, got %d", n_groups);
  b200::Counts c{{0, 0, 0}};
  for (int g = 0; g < n_groups; ++g) {
    B200_CHECK_ARG(counts[g] >= 1, "perceptual_mean: group %d is empty", g);
    c.n[g] = counts[g];
  }
  B200_CUDA(b200::launch_kernel(b200::perceptual_mean_kernel, dim3(1), dim3(1), 0, stream, image, (int)n_groups, c,
                                means, loss));
  B200_LAUNCH_CHECK("perceptual_mean_kernel");
  return B200_OK;
}
