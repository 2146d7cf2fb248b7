// Shared helpers for libb200gen.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <stdlib.h>
#include <utility>
#include "../../include/b200gen.h"

namespace b200 {

// thread-local last-error text, set by every failing entry point
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define B200_CHECK_ARG(cond, ...)                    \
  do {                                               \
    if (!(cond)) {                                   \
      b200::set_error(__VA_ARGS__);                  \
      return B200_EINVAL;                            \
    }                                                \
  } while (0)

#define B200_CUDA(call)                                              \
  do {                                                               \
    cudaError_t e__ = (call);                                        \
    if (e__ != cudaSuccess) return b200::cuda_fail(e__, #call);      \
  } while (0)

#define B200_LAUNCH_CHECK(name)                                      \
  do {                                                               \
    cudaError_t e__ = cudaGetLastError();                            \
    if (e__ != cudaSuccess) return b200::cuda_fail(e__, name);       \
  } while (0)

int sm_count();

// Every kernel of the library goes out through this: launch_kernel(k, grid, block, smem, stream, args...), or
// launch_kernel<Cluster>(...) for a kernel that runs in thread-block clusters of Cluster CTAs along x.
template <int Cluster = 1, typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  if (Cluster > 1) {
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = Cluster;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == B200_ACT_RELU) return fmaxf(x, 0.0f);
  if (act == B200_ACT_SILU) return silu_f(x);
  if (act == B200_ACT_LEAKYRELU) return x > 0.0f ? x : 0.01f * x;
  if (act == B200_ACT_LEAKYRELU02) return x > 0.0f ? x : 0.2f * x;
  if (act == B200_ACT_GELU) return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
  if (act == B200_ACT_TANH) return tanhf(x);
  if (act == B200_ACT_SIGMOID) return 1.0f / (1.0f + __expf(-x));
  return x;
}

// ------------------------------------------------------------------------------------------------
// The library's 16-bit storage type ("h16") for activations and packed weights.  Default: IEEE fp16 — 11 significand
// bits against bfloat16's 8, at the same wgmma rate and the same bytes; the reference-generated C2
// fixture (DESIGN.md section 3) needs the extra bits: an all-bf16 data path is 7.9e-2 off the fp32 reference at its
// ill-conditioned probe, an all-fp16 one 7.8e-3.  fp32 -> fp16 conversions saturate (F2FP.SATFINITE: +-65504 instead
// of inf), so an out-of-range activation degrades instead of poisoning the sample with NaNs.
// -DB200_H16_IS_BF16 builds the bfloat16 flavour (libb200gen_bf16.so) for models whose activations exceed fp16's range.
// ------------------------------------------------------------------------------------------------
#ifdef B200_H16_IS_BF16
typedef __nv_bfloat16 h16;
typedef __nv_bfloat162 h162;
#define B200_H16_TMAP CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
#define B200_H16_NAME "bf16"
__device__ __forceinline__ h16 f2h(float x) { return __float2bfloat16_rn(x); }
__device__ __forceinline__ float h2f(h16 x) { return __bfloat162float(x); }
__device__ __forceinline__ h162 f2h2(float a, float b) { return __floats2bfloat162_rn(a, b); }
__device__ __forceinline__ float2 h22f2(h162 v) { return __bfloat1622float2(v); }
#else
typedef __half h16;
typedef __half2 h162;
#define B200_H16_TMAP CU_TENSOR_MAP_DATA_TYPE_FLOAT16
#define B200_H16_NAME "fp16"
__device__ __forceinline__ h162 f2h2(float a, float b) {  // low half = a, high half = b; saturating
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return *reinterpret_cast<h162*>(&r);
}
__device__ __forceinline__ h16 f2h(float x) {
  unsigned short r;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(x));
  return *reinterpret_cast<h16*>(&r);
}
__device__ __forceinline__ float h2f(h16 x) { return __half2float(x); }
__device__ __forceinline__ float2 h22f2(h162 v) { return __half22float2(v); }
#endif

// 8 h16 <-> 8 floats through one 16-byte vector
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const h162* h = reinterpret_cast<const h162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = h22f2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 v;
  h162* h = reinterpret_cast<h162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = f2h2(f[2 * i], f[2 * i + 1]);
  return v;
}

// element i of an fp32 / fp64 / IEEE fp16 / bf16 array (B200_DT_F32 / _F64 / _FP16 / _BF16) as fp32
__device__ __forceinline__ float load_any(const void* p, int dt, int64_t i) {
  switch (dt) {
    case B200_DT_F32: return static_cast<const float*>(p)[i];
    case B200_DT_F64: return static_cast<float>(static_cast<const double*>(p)[i]);
    case B200_DT_FP16: return __half2float(static_cast<const __half*>(p)[i]);
    default: return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
  }
}
// the same element as fp64 (exact for every format)
__device__ __forceinline__ double load_any_f64(const void* p, int dt, int64_t i) {
  return dt == B200_DT_F64 ? static_cast<const double*>(p)[i] : static_cast<double>(load_any(p, dt, i));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace b200
