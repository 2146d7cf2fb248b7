// HBM-bound helpers of the sampling path: layout conversion on the API edge, resampling, GEGLU, row softmax,
// time embedding, GEMV-class linears and the fused scheduler updates.  All are single-pass, coalesced and
// (where the layout allows) 128-bit vectorised; none of them has data reuse worth staging in shared memory
// except the two transposes.
#include "common.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------
// NC[D]HW fp32 <-> NDHWC bf16: 32x32 shared-memory tile transpose (coalesced on both sides).
// ------------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int C, long long spatial,
                                    h16* __restrict__ y, int pitch) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long s0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const float* xb = x + (long long)n * C * spatial;
  h16* yb = y + (long long)n * spatial * pitch;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j;
    const long long s = s0 + threadIdx.x;
    tile[j][threadIdx.x] = (c < C && s < spatial) ? xb[(long long)c * spatial + s] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const long long s = s0 + j;
    const int c = c0 + threadIdx.x;
    if (s < spatial && c < pitch) yb[s * pitch + c] = f2h(tile[threadIdx.x][j]);
  }
}

template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ x, int C, long long spatial, int pitch,
                                    float* __restrict__ y) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long s0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const T* xb = x + (long long)n * spatial * pitch;
  float* yb = y + (long long)n * C * spatial;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const long long s = s0 + j;
    const int c = c0 + threadIdx.x;
    float v = 0.f;
    if (s < spatial && c < C) {
      if constexpr (sizeof(T) == 2) v = h2f(xb[s * pitch + c]);
      else v = xb[s * pitch + c];
    }
    tile[j][threadIdx.x] = v;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j;
    const long long s = s0 + threadIdx.x;
    if (c < C && s < spatial) yb[(long long)c * spatial + s] = tile[threadIdx.x][j];
  }
}

// ------------------------------------------------------------------------------------------------
// x2 bilinear / bicubic upsample of a 2-D channels-last tensor (align_corners=False); one thread per (output pixel,
// 8 channels).  Output o = 2i + parity reads source coordinate s = i - 0.25 (even) or i + 0.25 (odd), so each axis has
// two sets of taps and weights, picked by parity.
// ------------------------------------------------------------------------------------------------
// bilinear: s clamped at 0 (only the first even output is affected: it copies row 0)
__device__ __forceinline__ void interp_taps_linear(int o, int n, int* idx, float* w) {
  const int i = o >> 1;
  if (o & 1)       { idx[0] = i;     idx[1] = min(i + 1, n - 1); w[0] = 0.75f; w[1] = 0.25f; }
  else if (i == 0) { idx[0] = 0;     idx[1] = 0;                 w[0] = 1.0f;  w[1] = 0.0f;  }
  else             { idx[0] = i - 1; idx[1] = i;                 w[0] = 0.25f; w[1] = 0.75f; }
}
// bicubic: upsample_bicubic2d's cubic convolution (A = -0.75) at fraction t = 0.75 (even) or 0.25 (odd), taps
// floor(s) - 1 .. floor(s) + 2 clamped to the border
__device__ __forceinline__ void interp_taps_cubic(int o, int n, int* idx, float* w) {
  const float A = -0.75f;
  const int f = (o & 1) ? (o >> 1) : (o >> 1) - 1;
  const float t = (o & 1) ? 0.25f : 0.75f;
  const float x0 = t + 1.0f, x1 = t, x2 = 1.0f - t, x3 = 2.0f - t;
  w[0] = ((A * x0 - 5.0f * A) * x0 + 8.0f * A) * x0 - 4.0f * A;
  w[1] = ((A + 2.0f) * x1 - (A + 3.0f)) * x1 * x1 + 1.0f;
  w[2] = ((A + 2.0f) * x2 - (A + 3.0f)) * x2 * x2 + 1.0f;
  w[3] = ((A * x3 - 5.0f * A) * x3 + 8.0f * A) * x3 - 4.0f * A;
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = min(max(f - 1 + k, 0), n - 1);
}

template <int MODE>
__global__ void upsample2x_interp_kernel(const uint4* __restrict__ x, int N, int H, int W, int pv,
                                         uint4* __restrict__ y) {
  constexpr int T = MODE == B200_INTERP_BICUBIC ? 4 : 2;
  const int OH = 2 * H, OW = 2 * W;
  const long long total = (long long)N * OH * OW * pv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int v = (int)(t % pv); t /= pv;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH); t /= OH;
    const int n = (int)t;
    int hi[T], wi[T];
    float hw[T], ww[T];
    if constexpr (MODE == B200_INTERP_BICUBIC) {
      interp_taps_cubic(oh, H, hi, hw);
      interp_taps_cubic(ow, W, wi, ww);
    } else {
      interp_taps_linear(oh, H, hi, hw);
      interp_taps_linear(ow, W, wi, ww);
    }
    const uint4* img = x + (long long)n * H * W * pv + v;
    float out[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) out[c] = 0.f;
#pragma unroll
    for (int a = 0; a < T; ++a) {            // interpolate along W within each source row, then along H
      float row[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) row[c] = 0.f;
#pragma unroll
      for (int b = 0; b < T; ++b) {
        float f[8];
        unpack8(__ldg(img + ((long long)hi[a] * W + wi[b]) * pv), f);
#pragma unroll
        for (int c = 0; c < 8; ++c) row[c] = fmaf(f[c], ww[b], row[c]);
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) out[c] = fmaf(row[c], hw[a], out[c]);
    }
    y[idx] = pack8(out);
  }
}

// ------------------------------------------------------------------------------------------------
// k^dims window, stride 2, padding p on channels-last h16 (PatchGAN pyramid pooling); one thread per (output voxel,
// 8 channels).  Avg counts the padding (count_include_pad=True: with floor-mode output sizes every window lies inside
// the padded extent, so the divisor is k^dims); max skips it (-inf) and keeps the first NaN it meets, like PyTorch.
// ------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void pool_s2_kernel(const uint4* __restrict__ x, int N, int D, int H, int W, int pv, int dims, int k,
                               int pad, int OD, int OH, int OW, uint4* __restrict__ y) {
  const int kd = dims == 3 ? k : 1;
  const float div = (float)(kd * k * k);
  const long long total = (long long)N * OD * OH * OW * pv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int v = (int)(t % pv); t /= pv;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH); t /= OH;
    const int od = (int)(t % OD); t /= OD;
    const int n = (int)t;
    const int d0 = dims == 3 ? od * 2 - pad : od, h0 = oh * 2 - pad, w0 = ow * 2 - pad;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = MODE == B200_POOL_MAX ? -INFINITY : 0.f;
    for (int a = 0; a < kd; ++a) {
      const int id = d0 + a;
      if (id < 0 || id >= D) continue;
      for (int b = 0; b < k; ++b) {
        const int ih = h0 + b;
        if (ih < 0 || ih >= H) continue;
        const uint4* row = x + (((long long)n * D + id) * H + ih) * W * pv + v;
        for (int c = 0; c < k; ++c) {
          const int iw = w0 + c;
          if (iw < 0 || iw >= W) continue;
          float f[8];
          unpack8(__ldg(row + (long long)iw * pv), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if constexpr (MODE == B200_POOL_MAX) acc[j] = (f[j] > acc[j] || isnan(f[j])) ? f[j] : acc[j];
            else acc[j] += f[j];
          }
        }
      }
    }
    if constexpr (MODE == B200_POOL_AVG) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] /= div;
    }
    y[idx] = pack8(acc);
  }
}

// ------------------------------------------------------------------------------------------------
// F.interpolate(size | scale_factor, mode, align_corners=False) at any size, on any strided layout; the coordinate
// rules are ATen's (include/b200gen.h, b200_interpolate).  FAM picks the kernel family, V the thread mapping:
//   V = 8: one thread per (output voxel, 8 channels), 16-byte vectors across channels (channel stride 1);
//   V = 1: one thread per output element, W fastest, so that planar reads and writes coalesce.
// The coordinate arithmetic spells out every rounding with _rn intrinsics (nearest indices depend on the exact
// rounding of dst * ratio).  Interpolation sums are separately rounded products and sums, left to right.
// ------------------------------------------------------------------------------------------------
enum { INTERP_FAM_NEAREST = 0, INTERP_FAM_LINEAR = 1, INTERP_FAM_CUBIC = 2, INTERP_FAM_AREA = 3 };

struct InterpArgs {
  const void* x;
  void* y;
  long long xs[5], ys[5];  // element strides n, c, d, h, w
  int x_dt, y_dt;
  int N, C, D, H, W, OD, OH, OW, dims;
  float rd, rh, rw;        // per-axis ratio (see the header)
};

template <int V>
__device__ __forceinline__ void interp_load(const void* x, int dt, long long off, float* f) {
  if constexpr (V == 8) {
    if (dt == B200_DT_H16) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const h16*>(x) + off)), f);
    } else {
      const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + off);
      const float4 a = __ldg(p), b = __ldg(p + 1);
      f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
      f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    }
  } else {
    f[0] = dt == B200_DT_H16   ? h2f(reinterpret_cast<const h16*>(x)[off])
           : dt == B200_DT_F32 ? __ldg(reinterpret_cast<const float*>(x) + off)
                               : load_any(x, dt, off);
  }
}

template <int V>
__device__ __forceinline__ void interp_store(void* y, int dt, long long off, const float* f) {
  if constexpr (V == 8) {
    if (dt == B200_DT_H16) {
      *reinterpret_cast<uint4*>(reinterpret_cast<h16*>(y) + off) = pack8(f);
    } else {
      float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + off);
      p[0] = make_float4(f[0], f[1], f[2], f[3]);
      p[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
  } else {
    if (dt == B200_DT_H16) reinterpret_cast<h16*>(y)[off] = f2h(f[0]);
    else reinterpret_cast<float*>(y)[off] = f[0];
  }
}

// nearest: min(floor(dst * ratio), in - 1), the product rounded once
__device__ __forceinline__ int interp_nearest(int o, int in, float r) {
  return min((int)floorf(__fmul_rn((float)o, r)), in - 1);
}

// source coordinate ratio * (dst + 0.5) - 0.5, one rounding (ATen's expression as compilers contract it)
__device__ __forceinline__ float interp_src(int o, float r) {
  return __fmaf_rn(r, __fadd_rn((float)o, 0.5f), -0.5f);
}

// linear: source clamped at 0; i0 = min(floor(s), in - 1), i1 = i0 + (i0 < in - 1), weights (1 - l, l) with
// l = clamp(s - i0, 0, 1); an axis whose extent does not change is copied (i0 = i1 = dst, weights (1, 0))
__device__ __forceinline__ void interp_taps_linear_any(int o, int in, int out, float r, int* i, float* w) {
  if (in == out) {
    i[0] = i[1] = o;
    w[0] = 1.f;
    w[1] = 0.f;
    return;
  }
  const float s = fmaxf(interp_src(o, r), 0.f);
  i[0] = min((int)floorf(s), in - 1);
  i[1] = i[0] + (i[0] < in - 1 ? 1 : 0);
  const float l = fminf(fmaxf(__fsub_rn(s, (float)i[0]), 0.f), 1.f);
  w[0] = __fsub_rn(1.f, l);
  w[1] = l;
}

// cubic (A = -0.75): source not clamped; f = min(floor(s), in - 1), t = clamp(s - f, 0, 1); taps f - 1 .. f + 2 each
// clamped to [0, in - 1]; weights cc2(t + 1), cc1(t), cc1(1 - t), cc2(2 - t) with
// cc1(x) = ((A + 2) x - (A + 3)) x x + 1 and cc2(x) = ((A x - 5A) x + 8A) x - 4A
// (Horner steps fused like the contracted ATen expressions)
__device__ __forceinline__ float interp_cc1(float x) {
  return __fmaf_rn(__fmul_rn(__fmaf_rn(1.25f, x, -2.25f), x), x, 1.f);
}
__device__ __forceinline__ float interp_cc2(float x) {
  return __fmaf_rn(__fmaf_rn(__fmaf_rn(-0.75f, x, 3.75f), x, -6.f), x, 3.f);
}
__device__ __forceinline__ void interp_taps_cubic_any(int o, int in, float r, int* i, float* w) {
  const float s = interp_src(o, r);
  const int f = min((int)floorf(s), in - 1);
  const float t = fminf(fmaxf(__fsub_rn(s, (float)f), 0.f), 1.f);
  const float u = __fsub_rn(1.f, t);
  w[0] = interp_cc2(__fadd_rn(t, 1.f));
  w[1] = interp_cc1(t);
  w[2] = interp_cc1(u);
  w[3] = interp_cc2(__fadd_rn(u, 1.f));
#pragma unroll
  for (int k = 0; k < 4; ++k) i[k] = min(max(f - 1 + k, 0), in - 1);
}

template <int FAM, int V>
__global__ void __launch_bounds__(256) interpolate_kernel(const InterpArgs a) {
  const int CG = V == 8 ? (a.C + 7) >> 3 : a.C;
  const long long total = (long long)a.N * CG * a.OD * a.OH * a.OW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    int cg = 0;
    if constexpr (V == 8) { cg = (int)(t % CG); t /= CG; }
    const int ow = (int)(t % a.OW); t /= a.OW;
    const int oh = (int)(t % a.OH); t /= a.OH;
    const int od = (int)(t % a.OD); t /= a.OD;
    if constexpr (V == 1) { cg = (int)(t % CG); t /= CG; }
    const long long n = t;
    const int c = V == 8 ? cg * 8 : cg;
    const long long xb = n * a.xs[0] + (long long)c * a.xs[1];
    float out[V];
    if constexpr (FAM == INTERP_FAM_NEAREST) {
      const int id = interp_nearest(od, a.D, a.rd), ih = interp_nearest(oh, a.H, a.rh),
                iw = interp_nearest(ow, a.W, a.rw);
      interp_load<V>(a.x, a.x_dt, xb + id * a.xs[2] + ih * a.xs[3] + iw * a.xs[4], out);
    } else if constexpr (FAM == INTERP_FAM_AREA) {
      // adaptive average: window [floor(o * in / out), ceil((o + 1) * in / out)) per axis, summed d, h, w
      // (innermost last), then divided by the three window extents in turn.  32-bit unsigned bounds (the entry point
      // checks in * out + out <= 2^32): a 64-bit division is a subroutine call the 8-channel kernel would spill around
      const unsigned D = a.D, H = a.H, W = a.W, OD = a.OD, OH = a.OH, OW = a.OW;
      const int d0 = (int)(od * D / OD), d1 = (int)(((od + 1) * D + OD - 1) / OD);
      const int h0 = (int)(oh * H / OH), h1 = (int)(((oh + 1) * H + OH - 1) / OH);
      const int w0 = (int)(ow * W / OW), w1 = (int)(((ow + 1) * W + OW - 1) / OW);
#pragma unroll
      for (int j = 0; j < V; ++j) out[j] = 0.f;
      for (int id = d0; id < d1; ++id)
        for (int ih = h0; ih < h1; ++ih) {
          const long long row = xb + id * a.xs[2] + ih * a.xs[3];
          for (int iw = w0; iw < w1; ++iw) {
            float f[V];
            interp_load<V>(a.x, a.x_dt, row + iw * a.xs[4], f);
#pragma unroll
            for (int j = 0; j < V; ++j) out[j] = __fadd_rn(out[j], f[j]);
          }
        }
#pragma unroll
      for (int j = 0; j < V; ++j)
        out[j] = __fdiv_rn(__fdiv_rn(__fdiv_rn(out[j], (float)(d1 - d0)), (float)(h1 - h0)), (float)(w1 - w0));
    } else {
      // separable: interpolate along W within each source row, then along H, then along D (dims 2 and 3)
      constexpr int T = FAM == INTERP_FAM_CUBIC ? 4 : 2;
      int wi[T], hi[T], di[2] = {od, od};
      float ww[T], hw[T], dw[2] = {1.f, 0.f};
#pragma unroll
      for (int k = 0; k < T; ++k) { hi[k] = oh; hw[k] = 0.f; }
      if constexpr (FAM == INTERP_FAM_CUBIC) {
        interp_taps_cubic_any(ow, a.W, a.rw, wi, ww);
        interp_taps_cubic_any(oh, a.H, a.rh, hi, hw);
      } else {
        interp_taps_linear_any(ow, a.W, a.OW, a.rw, wi, ww);
        if (a.dims >= 2) interp_taps_linear_any(oh, a.H, a.OH, a.rh, hi, hw);
        if (a.dims == 3) interp_taps_linear_any(od, a.D, a.OD, a.rd, di, dw);
      }
      const int TH = a.dims >= 2 ? T : 1, TD = a.dims == 3 ? 2 : 1;
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        if (p >= TD) break;
        float plane[V];
#pragma unroll
        for (int q = 0; q < T; ++q) {
          if (q >= TH) break;
          float row[V];
#pragma unroll
          for (int k = 0; k < T; ++k) {
            float f[V];
            interp_load<V>(a.x, a.x_dt, xb + di[p] * a.xs[2] + hi[q] * a.xs[3] + wi[k] * a.xs[4], f);
#pragma unroll
            for (int j = 0; j < V; ++j) row[j] = k == 0 ? __fmul_rn(f[j], ww[0]) : __fadd_rn(row[j], __fmul_rn(f[j], ww[k]));
          }
#pragma unroll
          for (int j = 0; j < V; ++j)
            plane[j] = TH == 1 ? row[j] : q == 0 ? __fmul_rn(row[j], hw[0]) : __fadd_rn(plane[j], __fmul_rn(row[j], hw[q]));
        }
#pragma unroll
        for (int j = 0; j < V; ++j)
          out[j] = TD == 1 ? plane[j] : p == 0 ? __fmul_rn(plane[j], dw[0]) : __fadd_rn(out[j], __fmul_rn(plane[j], dw[p]));
      }
    }
    interp_store<V>(a.y, a.y_dt, n * a.ys[0] + (long long)c * a.ys[1] + od * a.ys[2] + oh * a.ys[3] + ow * a.ys[4], out);
  }
}

__global__ void axpy_h16_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, float alpha,
                                 uint4* __restrict__ y, long long nvec) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec;
       idx += (long long)gridDim.x * blockDim.x) {
    float fa[8], fb[8];
    unpack8(__ldg(a + idx), fa);
    unpack8(__ldg(b + idx), fb);
#pragma unroll
    for (int j = 0; j < 8; ++j) fa[j] = fmaf(alpha, fb[j], fa[j]);
    y[idx] = pack8(fa);
  }
}

__global__ void copy_channels_kernel(const h16* __restrict__ src, int C, int src_pitch,
                                     h16* __restrict__ dst, int dst_pitch, int dst_off, long long rows, int vec) {
  const int per_row = C / vec;
  const long long total = rows * per_row;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / per_row;
    const int c = (int)(idx % per_row) * vec;
    if (vec == 8)
      *reinterpret_cast<uint4*>(dst + r * dst_pitch + dst_off + c) = __ldg(reinterpret_cast<const uint4*>(src + r * src_pitch + c));
    else
      dst[r * dst_pitch + dst_off + c] = src[r * src_pitch + c];
  }
}

// ------------------------------------------------------------------------------------------------
// GEGLU: y = x[:, :H] * gelu_erf(x[:, H:])
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

__global__ void geglu_kernel(const h16* __restrict__ x, long long M, int H, int x_pitch,
                             h16* __restrict__ y, int y_pitch) {
  const int HV = H / 8;
  const long long total = M * HV;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long m = idx / HV;
    const int h = (int)(idx % HV) * 8;
    float a[8], g[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + m * x_pitch + h)), a);
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + m * x_pitch + H + h)), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] *= gelu_erf(g[j]);
    *reinterpret_cast<uint4*>(y + m * y_pitch + h) = pack8(a);
  }
}

// ------------------------------------------------------------------------------------------------
// Row softmax: fp32 scores -> 16-bit probabilities.  The score GEMM's epilogue already left (max, sum exp) per
// 128-column tile of every row, so the row maximum and denominator come from a few hundred partials and the scores
// are read exactly once.
// ------------------------------------------------------------------------------------------------
__global__ void softmax_rows_partials_kernel(const float* __restrict__ s, int S, long long s_pitch,
                                             const float2* __restrict__ part, int n_tiles,
                                             h16* __restrict__ p, long long p_pitch) {
  const long long row = blockIdx.x;
  const int t = threadIdx.x;
  __shared__ float red[8];
  const float2* pr = part + row * n_tiles;
  float mx = -INFINITY;
  for (int i = t; i < n_tiles; i += 256) mx = fmaxf(mx, pr[i].x);
  mx = warp_max(mx);
  if ((t & 31) == 0) red[t >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = t; i < n_tiles; i += 256) {
    const float2 q = pr[i];
    if (q.x > -INFINITY) sum += q.y * __expf(q.x - mx);
  }
  sum = warp_sum(sum);
  if ((t & 31) == 0) red[t >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  const float* sr = s + row * s_pitch;
  h16* po = p + row * p_pitch;
  const bool vec = (s_pitch % 4 == 0) && (p_pitch % 4 == 0) && ((reinterpret_cast<uintptr_t>(s) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(p) & 7) == 0);
  if (vec) {
    const int S4 = S / 4;
    for (int c = t; c < S4; c += 256) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(sr) + c);
      h162 lo = f2h2(__expf(v.x - mx) * inv, __expf(v.y - mx) * inv);
      h162 hi = f2h2(__expf(v.z - mx) * inv, __expf(v.w - mx) * inv);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&lo);
      o.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(po + 4 * (long long)c) = o;
    }
    for (int c = S4 * 4 + t; c < S; c += 256) po[c] = f2h(__expf(sr[c] - mx) * inv);
  } else {
    for (int c = t; c < S; c += 256) po[c] = f2h(__expf(sr[c] - mx) * inv);
  }
  for (long long c = S + t; c < p_pitch; c += 256) po[c] = f2h(0.f);
}

// ------------------------------------------------------------------------------------------------
// time embedding + GEMV-class linear
// ------------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int N, int dim, float max_period,
                                          float* __restrict__ emb) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * dim) return;
  const int n = idx / dim, i = idx % dim;
  float v = 0.f;
  if (i < 2 * half) {
    const int k = i < half ? i : i - half;
    // exponent = -ln(max_period) * k, freq = exp(exponent / half): same operation order as the reference
    const float freq = expf((-logf(max_period) * (float)k) / (float)half);
    const float arg = t[n] * freq;
    v = i < half ? cosf(arg) : sinf(arg);
  }
  emb[idx] = v;
}

// one warp per output feature; loops over the (few) rows.  VEC: K % 128 == 0 and 16-byte aligned rows — every lane
// issues all its float4 weight loads before the first FMA (a time-embedding projection is one 4 KB row per warp: the
// scalar form waits on 32 dependent-latency loads).
template <bool VEC>
__global__ void small_linear_kernel(const float* __restrict__ x, int M, int K, const float* __restrict__ W,
                                    const float* __restrict__ b, int O, int act_in, int act_out,
                                    float* __restrict__ y) {
  const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (o >= O) return;
  const int lane = threadIdx.x & 31;
  const float* w = W + (long long)o * K;
  for (int m = 0; m < M; ++m) {
    const float* xr = x + (long long)m * K;
    float acc = 0.f;
    if constexpr (VEC) {
      for (int k0 = 0; k0 < K; k0 += 1024) {
        float4 wv[8], xv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k = k0 + i * 128 + lane * 4;
          if (k < K) {
            wv[i] = __ldg(reinterpret_cast<const float4*>(w + k));
            xv[i] = *reinterpret_cast<const float4*>(xr + k);
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (k0 + i * 128 + lane * 4 < K) {
            acc = fmaf(apply_act(xv[i].x, act_in), wv[i].x, acc);
            acc = fmaf(apply_act(xv[i].y, act_in), wv[i].y, acc);
            acc = fmaf(apply_act(xv[i].z, act_in), wv[i].z, acc);
            acc = fmaf(apply_act(xv[i].w, act_in), wv[i].w, acc);
          }
        }
      }
    } else {
      for (int k = lane; k < K; k += 32) acc = fmaf(apply_act(xr[k], act_in), __ldg(w + k), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) y[(long long)m * O + o] = apply_act(acc + (b ? b[o] : 0.f), act_out);
  }
}

// ------------------------------------------------------------------------------------------------
// scheduler steps
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ddim_one(const b200_ddim_coef& c, float m, float s, float nz, bool has_noise, float& p,
                                         float& x0) {
  float eps;
  if (c.prediction_type == B200_PRED_EPSILON) {
    x0 = (s - c.sqrt_beta_prod_t * m) / c.sqrt_alpha_prod_t;
    eps = m;
  } else if (c.prediction_type == B200_PRED_SAMPLE) {
    x0 = m;
    eps = (s - c.sqrt_alpha_prod_t * x0) / c.sqrt_beta_prod_t;
  } else {
    x0 = c.sqrt_alpha_prod_t * s - c.sqrt_beta_prod_t * m;
    eps = c.sqrt_alpha_prod_t * m + c.sqrt_beta_prod_t * s;
  }
  if (c.clip) x0 = fminf(fmaxf(x0, c.clip_min), c.clip_max);
  p = c.sqrt_alpha_prod_prev * x0 + c.dir_coef * eps;
  if (has_noise) p += c.sigma * nz;
}

// 128-bit loads / stores, two independent vectors per thread and iteration (the update is 2 reads + 2 writes of 4 B per
// element: pure HBM streaming, so what matters is bytes in flight per SM); scalar tail for n % 4.
// VEC = 0: pointers not 16-byte aligned -> scalar path.
template <int VEC>
__global__ void __launch_bounds__(256) ddim_step_kernel(const float* __restrict__ eps_in, const float* __restrict__ x,
                                                        const float* __restrict__ noise, b200_ddim_coef c,
                                                        float* __restrict__ prev, float* __restrict__ x0_out, long long n) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
  const bool has_noise = noise != nullptr;
  long long done = 0;
  if (VEC) {
    const long long nv = n >> 2;
    const float4* e4 = reinterpret_cast<const float4*>(eps_in);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* n4 = reinterpret_cast<const float4*>(noise);
    float4* p4 = reinterpret_cast<float4*>(prev);
    float4* o4 = reinterpret_cast<float4*>(x0_out);
    for (long long i = tid; i < nv; i += 2 * nthr) {
      const long long i2 = i + nthr;
      const bool two = i2 < nv;
      const float4 ma = __ldg(e4 + i), sa = __ldg(x4 + i);
      const float4 mb = two ? __ldg(e4 + i2) : ma, sb = two ? __ldg(x4 + i2) : sa;
      float4 za = make_float4(0.f, 0.f, 0.f, 0.f), zb = za;
      if (has_noise) { za = __ldg(n4 + i); if (two) zb = __ldg(n4 + i2); }
      float4 pa, oa, pb, ob;
      ddim_one(c, ma.x, sa.x, za.x, has_noise, pa.x, oa.x); ddim_one(c, ma.y, sa.y, za.y, has_noise, pa.y, oa.y);
      ddim_one(c, ma.z, sa.z, za.z, has_noise, pa.z, oa.z); ddim_one(c, ma.w, sa.w, za.w, has_noise, pa.w, oa.w);
      ddim_one(c, mb.x, sb.x, zb.x, has_noise, pb.x, ob.x); ddim_one(c, mb.y, sb.y, zb.y, has_noise, pb.y, ob.y);
      ddim_one(c, mb.z, sb.z, zb.z, has_noise, pb.z, ob.z); ddim_one(c, mb.w, sb.w, zb.w, has_noise, pb.w, ob.w);
      p4[i] = pa;
      if (x0_out) o4[i] = oa;
      if (two) { p4[i2] = pb; if (x0_out) o4[i2] = ob; }
    }
    done = nv << 2;
  }
  for (long long i = done + tid; i < n; i += nthr) {
    float p, x0;
    ddim_one(c, eps_in[i], x[i], has_noise ? noise[i] : 0.f, has_noise, p, x0);
    prev[i] = p;
    if (x0_out) x0_out[i] = x0;
  }
}

__global__ void ddpm_step_kernel(const float* __restrict__ eps_in, const float* __restrict__ x,
                                 const float* __restrict__ noise, const float* __restrict__ pred_var,
                                 b200_ddpm_coef c, float* __restrict__ prev, float* __restrict__ x0_out,
                                 long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float m = eps_in[i], s = x[i];
    float x0;
    if (c.prediction_type == B200_PRED_EPSILON) x0 = (s - c.sqrt_beta_prod_t * m) / c.sqrt_alpha_prod_t;
    else if (c.prediction_type == B200_PRED_SAMPLE) x0 = m;
    else x0 = c.sqrt_alpha_prod_t * s - c.sqrt_beta_prod_t * m;
    if (c.clip) x0 = fminf(fmaxf(x0, c.clip_min), c.clip_max);
    float p = c.coef_x0 * x0 + c.coef_xt * s;
    if (noise) {
      float sig = c.sigma;
      if (c.var_mode == 1) sig = sqrtf(pred_var[i]);
      else if (c.var_mode == 2) {
        const float frac = (pred_var[i] + 1.0f) / 2.0f;
        sig = sqrtf(frac * c.max_log + (1.0f - frac) * c.min_log);
      }
      p += sig * noise[i];
    }
    prev[i] = p;
    if (x0_out) x0_out[i] = x0;
  }
}

// tanh approximation of the standard normal CDF used by the reference (inferer.py:279-283)
__device__ __forceinline__ float approx_normal_cdf(float x) {
  return 0.5f * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

__global__ void ddpm_kl_kernel(const float* __restrict__ x0, const float* __restrict__ xt,
                               const float* __restrict__ mo, b200_kl_coef c, float* __restrict__ kl_out,
                               double* __restrict__ sample_sum, long long per_sample) {
  const int n = blockIdx.y;
  const long long base = (long long)n * per_sample;
  double acc = 0.0;                             // fp64 per thread: a thread sums per_sample / (grid threads) terms
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_sample;
       i += (long long)gridDim.x * blockDim.x) {
    const float a = x0[base + i], s = xt[base + i], m = mo[base + i];
    float p0;
    if (c.prediction_type == B200_PRED_EPSILON) p0 = (s - c.sqrt_beta_prod_t * m) / c.sqrt_alpha_prod_t;
    else if (c.prediction_type == B200_PRED_SAMPLE) p0 = m;
    else p0 = c.sqrt_alpha_prod_t * s - c.sqrt_beta_prod_t * m;
    if (c.clip) p0 = fminf(fmaxf(p0, -1.0f), 1.0f);
    const float pred_mean = c.coef_x0 * p0 + c.coef_xt * s;
    float kl;
    if (c.is_t0) {
      // -log p(x_0 | x_1): discretised Gaussian (inferer.py:285-321)
      const float centered = a - pred_mean;
      const float inv_stdv = expf(-0.5f * c.log_pred_var);
      const float cdf_plus = approx_normal_cdf(inv_stdv * (centered + c.bin_width / 2));
      const float cdf_min = approx_normal_cdf(inv_stdv * (centered - c.bin_width / 2));
      float lp;
      if (a < -0.999f) lp = logf(fmaxf(cdf_plus, 1e-12f));
      else if (a > 0.999f) lp = logf(fmaxf(1.0f - cdf_min, 1e-12f));
      else lp = logf(fmaxf(cdf_plus - cdf_min, 1e-12f));
      kl = -lp;
    } else {
      const float post_mean = c.coef_x0 * a + c.coef_xt * s;
      const float d = post_mean - pred_mean;
      kl = 0.5f * (-1.0f + c.log_pred_var - c.log_post_var + expf(c.log_post_var - c.log_pred_var) +
                   d * d * expf(-c.log_pred_var));
    }
    if (kl_out) kl_out[base + i] = kl;
    acc += (double)kl;
  }
  __shared__ double red[8];
  double d = acc;
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    atomicAdd(sample_sum + n, t);
  }
}

struct PndmPtrs { const float* h[4]; };

__global__ void pndm_step_kernel(PndmPtrs hp, const float* __restrict__ x, b200_pndm_coef c,
                                 float* __restrict__ prev, float* __restrict__ eps_out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float e = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < c.n_hist) e = fmaf(c.w[k], hp.h[k][i], e);
    if (eps_out) eps_out[i] = e;
    if (prev) {
      const float s = x[i];
      if (c.prediction_type == B200_PRED_V) e = c.v_alpha * e + c.v_beta * s;
      prev[i] = c.sample_coeff * s - c.eps_coeff * e;
    }
  }
}

__global__ void add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                 const float* __restrict__ ca, const float* __restrict__ cb, float sign_b,
                                 long long per_sample, float* __restrict__ out) {
  const int n = blockIdx.y;
  const float a = ca[n], b = cb[n] * sign_b;
  const long long base = (long long)n * per_sample;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_sample;
       i += (long long)gridDim.x * blockDim.x)
    out[base + i] = a * x0[base + i] + b * noise[base + i];
}

__global__ void exp_half_clamped_kernel(const float* __restrict__ x, float lo, float hi, float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = expf(fminf(fmaxf(x[i], lo), hi) / 2.0f);
}

__global__ void fma_f32_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                               float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = a[i] + b[i] * c[i];
}

// one CTA: z elementwise, the KL sum in fp64 in a fixed order (strided per thread, then a fixed shuffle / shared tree)
__global__ void __launch_bounds__(256) vae_reparam_kld_kernel(const float* __restrict__ mu,
                                                              const float* __restrict__ logvar,
                                                              const float* __restrict__ eps, float* __restrict__ z,
                                                              float* __restrict__ kld, long long n) {
  double s = 0.0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float m = mu[i], lv = logvar[i];
    z[i] = fmaf(eps[i], expf(0.5f * lv), m);
    s += 1.0 + (double)lv - (double)m * (double)m - exp((double)lv);
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __shared__ double red[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
    kld[0] = (float)(-0.5 * t);
  }
}

__global__ void scale_f32_kernel(const float* __restrict__ x, float mul, float div, float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = x[i] * mul / div;
}

static unsigned grid_for(long long work, int threads = 256, int waves = 8) {
  long long b = (work + threads - 1) / threads;
  const long long cap = (long long)waves * sm_count();
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}


// ------------------------------------------------------------------------------------------------
// Tap reformulations of the two degenerate convolutions of the UNet (conv_in: 1 -> C, out: C -> 1): both are
// HBM-bound, but as 27-tap implicit GEMMs they pad K (or N) 2-60x.  tap_gather builds the tiny im2col matrix
// X2[v][tap * Cin + c] so that conv_in becomes ONE 64-wide K chunk; tap_sum evaluates
// out[v][co] = b[co] + sum_tap Y[v + off(tap)][tap * Cout + co] after a 1x1x1 GEMM Y = x W2^T that reads x once.
// ------------------------------------------------------------------------------------------------
struct TapGeom {
  int N, D, H, W, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw;
};

__global__ void tap_gather_kernel(const h16* __restrict__ x, int C, int x_pitch, TapGeom g,
                                  h16* __restrict__ out, int out_pitch) {
  // one thread per (output voxel, 8-column vector): the voxel coordinates are decoded once, the row is written with
  // 16-byte stores (out_pitch is a multiple of 8: it is the K pitch of the GEMM that follows)
  const int taps = g.kd * g.kh * g.kw;
  const int vecs = out_pitch >> 3;
  const long long total = (long long)g.N * g.OD * g.OH * g.OW * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v8 = (int)(i % vecs);
    long long v = i / vecs;
    const int ow = (int)(v % g.OW); long long t = v / g.OW;
    const int oh = (int)(t % g.OH); t /= g.OH;
    const int od = (int)(t % g.OD); const int n = (int)(t / g.OD);
    const h16* xn = x + (long long)n * g.D * g.H * g.W * x_pitch;
    __align__(16) h16 vals[8];
    int col = v8 * 8;
    int tap = col / C, c = col - tap * C;
#pragma unroll
    for (int e = 0; e < 8; ++e, ++col) {
      h16 val = f2h(0.f);
      if (tap < taps) {
        const int cw = tap % g.kw, bh = (tap / g.kw) % g.kh, ad = tap / (g.kw * g.kh);
        const int iw = ow * g.sw + cw - g.pw, ih = oh * g.sh + bh - g.ph, id = od * g.sd + ad - g.pd;
        if (iw >= 0 && iw < g.W && ih >= 0 && ih < g.H && id >= 0 && id < g.D)
          val = xn[(((long long)id * g.H + ih) * g.W + iw) * x_pitch + c];
      }
      vals[e] = val;
      if (++c == C) { c = 0; ++tap; }
    }
    *reinterpret_cast<uint4*>(out + v * out_pitch + v8 * 8) = *reinterpret_cast<const uint4*>(vals);
  }
}

template <int COUT>
__global__ void tap_sum_kernel(const float* __restrict__ y, int y_pitch, TapGeom g, const float* __restrict__ bias,
                               void* __restrict__ out, int out_pitch, int out_dtype) {
  const long long total = (long long)g.N * g.OD * g.OH * g.OW;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < total;
       v += (long long)gridDim.x * blockDim.x) {
    const int ow = (int)(v % g.OW); long long t = v / g.OW;
    const int oh = (int)(t % g.OH); t /= g.OH;
    const int od = (int)(t % g.OD); const int n = (int)(t / g.OD);
    float acc[COUT];
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = bias ? bias[co] : 0.f;
    for (int a = 0; a < g.kd; ++a) {
      const int id = od + a - g.pd;
      if (id < 0 || id >= g.D) continue;
      for (int b = 0; b < g.kh; ++b) {
        const int ih = oh + b - g.ph;
        if (ih < 0 || ih >= g.H) continue;
        const float* row = y + (((long long)n * g.D + id) * g.H + ih) * g.W * y_pitch + ((a * g.kh + b) * g.kw) * COUT;
#pragma unroll 3
        for (int c = 0; c < g.kw; ++c) {
          const int iw = ow + c - g.pw;
          if (iw < 0 || iw >= g.W) continue;
          const float* src = row + (long long)iw * y_pitch + c * COUT;
#pragma unroll
          for (int co = 0; co < COUT; ++co) acc[co] += __ldg(src + co);
        }
      }
    }
    if (out_dtype == B200_DT_H16) {
      h16* o = reinterpret_cast<h16*>(out) + v * out_pitch;
      for (int co = 0; co < out_pitch; ++co) o[co] = f2h(co < COUT ? acc[co < COUT ? co : 0] : 0.f);
    } else {
      float* o = reinterpret_cast<float*>(out) + v * out_pitch;
      for (int co = 0; co < out_pitch; ++co) o[co] = co < COUT ? acc[co < COUT ? co : 0] : 0.f;
    }
  }
}


// token + absolute position embedding rows -> bf16 (nets/transformer.py:97-99)
__global__ void embed_tokens_kernel(const long long* __restrict__ tokens, long long M, int seq_len, int pos0,
                                    const float* __restrict__ tok_emb, const float* __restrict__ pos_emb, int C,
                                    h16* __restrict__ out, int pitch, const int* __restrict__ pos_dev) {
  if (pos_dev) pos0 = *pos_dev;
  const long long total = M * pitch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % pitch);
    const long long m = i / pitch;
    float v = 0.f;
    if (c < C) v = tok_emb[tokens[m] * C + c] + pos_emb[(long long)(pos0 + (int)(m % seq_len)) * C + c];
    out[i] = f2h(v);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_nchw_to_nhwc(const float* x, int32_t N, int32_t C, int64_t spatial, void* y, int32_t pitch,
                                 void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && N >= 1 && C >= 1 && spatial >= 1 && pitch >= C, "nchw_to_nhwc: bad arguments");
  const long long bx = (spatial + 31) / 32;
  B200_CHECK_ARG(bx < (1ll << 31) && N <= 65535, "nchw_to_nhwc: extent too large");
  dim3 grid((unsigned)bx, (pitch + 31) / 32, N);
  B200_CUDA(b200::launch_kernel(nchw_to_nhwc_kernel, grid, dim3(32, 8), 0, stream, x, C, spatial, reinterpret_cast<h16*>(y), pitch));
  B200_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return B200_OK;
}

extern "C" int b200_nhwc_to_nchw(const void* x, int32_t x_dtype, int32_t N, int32_t C, int64_t spatial,
                                 int32_t pitch, float* y, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && N >= 1 && C >= 1 && spatial >= 1 && pitch >= C, "nhwc_to_nchw: bad arguments");
  const long long bx = (spatial + 31) / 32;
  B200_CHECK_ARG(bx < (1ll << 31) && N <= 65535, "nhwc_to_nchw: extent too large");
  dim3 grid((unsigned)bx, (C + 31) / 32, N);
  if (x_dtype == B200_DT_H16)
    B200_CUDA(b200::launch_kernel(nhwc_to_nchw_kernel<h16>, grid, dim3(32, 8), 0, stream, reinterpret_cast<const h16*>(x), C, spatial, pitch, y));
  else
    B200_CUDA(b200::launch_kernel(nhwc_to_nchw_kernel<float>, grid, dim3(32, 8), 0, stream, reinterpret_cast<const float*>(x), C, spatial, pitch, y));
  B200_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return B200_OK;
}

extern "C" int b200_upsample2x_interp(const void* x, int32_t N, int32_t H, int32_t W, int32_t pitch, int32_t mode,
                                      void* y, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && N >= 1 && H >= 1 && W >= 1 && pitch >= 8 && pitch % 8 == 0 &&
                 (uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0, "upsample2x_interp: bad arguments");
  B200_CHECK_ARG(mode == B200_INTERP_BILINEAR || mode == B200_INTERP_BICUBIC, "upsample2x_interp: unknown mode %d", mode);
  const long long total = (long long)N * 2 * H * 2 * W * (pitch / 8);
  if (mode == B200_INTERP_BICUBIC)
    B200_CUDA(b200::launch_kernel(upsample2x_interp_kernel<B200_INTERP_BICUBIC>, grid_for(total), 256, 0, stream,
                               reinterpret_cast<const uint4*>(x), N, H, W, pitch / 8, reinterpret_cast<uint4*>(y)));
  else
    B200_CUDA(b200::launch_kernel(upsample2x_interp_kernel<B200_INTERP_BILINEAR>, grid_for(total), 256, 0, stream,
                               reinterpret_cast<const uint4*>(x), N, H, W, pitch / 8, reinterpret_cast<uint4*>(y)));
  B200_LAUNCH_CHECK("upsample2x_interp_kernel");
  return B200_OK;
}

extern "C" int b200_vae_reparam_kld(const float* mu, const float* logvar, const float* eps, float* z, float* kld,
                                    int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(mu && logvar && eps && z && kld && n >= 1, "vae_reparam_kld: bad arguments");
  B200_CUDA(b200::launch_kernel(vae_reparam_kld_kernel, 1, 256, 0, stream, mu, logvar, eps, z, kld, (long long)n));
  B200_LAUNCH_CHECK("vae_reparam_kld_kernel");
  return B200_OK;
}

extern "C" int b200_pool_s2(const void* x, int32_t N, int32_t D, int32_t H, int32_t W, int32_t pitch, int32_t dims,
                            int32_t kernel, int32_t padding, int32_t mode, void* y, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && N >= 1 && D >= 1 && H >= 1 && W >= 1 && pitch >= 8 && pitch % 8 == 0 &&
                 (dims == 2 || dims == 3) && (uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0,
                 "pool_s2: bad arguments");
  B200_CHECK_ARG(mode == B200_POOL_AVG || mode == B200_POOL_MAX, "pool_s2: unknown mode %d", mode);
  B200_CHECK_ARG(kernel >= 1 && kernel <= 64 && padding >= 0 && 2 * padding <= kernel,
                 "pool_s2: kernel %d / padding %d (padding must be at most half the kernel)", kernel, padding);
  B200_CHECK_ARG(H + 2 * padding >= kernel && W + 2 * padding >= kernel && (dims == 2 || D + 2 * padding >= kernel),
                 "pool_s2: input %d x %d x %d smaller than the kernel %d with padding %d", D, H, W, kernel, padding);
  const int OD = dims == 3 ? (D + 2 * padding - kernel) / 2 + 1 : D;
  const int OH = (H + 2 * padding - kernel) / 2 + 1, OW = (W + 2 * padding - kernel) / 2 + 1;
  const long long total = (long long)N * OD * OH * OW * (pitch / 8);
  if (mode == B200_POOL_MAX)
    B200_CUDA(b200::launch_kernel(pool_s2_kernel<B200_POOL_MAX>, grid_for(total), 256, 0, stream,
                               reinterpret_cast<const uint4*>(x), N, D, H, W, pitch / 8, dims, kernel, padding, OD, OH,
                               OW, reinterpret_cast<uint4*>(y)));
  else
    B200_CUDA(b200::launch_kernel(pool_s2_kernel<B200_POOL_AVG>, grid_for(total), 256, 0, stream,
                               reinterpret_cast<const uint4*>(x), N, D, H, W, pitch / 8, dims, kernel, padding, OD, OH,
                               OW, reinterpret_cast<uint4*>(y)));
  B200_LAUNCH_CHECK("pool_s2_kernel");
  return B200_OK;
}

template <int FAM>
static cudaError_t launch_interpolate(const b200::InterpArgs& a, bool vec, cudaStream_t stream) {
  const long long total = (long long)a.N * (vec ? (a.C + 7) / 8 : a.C) * a.OD * a.OH * a.OW;
  if (vec) return b200::launch_kernel(interpolate_kernel<FAM, 8>, grid_for(total), 256, 0, stream, a);
  return b200::launch_kernel(interpolate_kernel<FAM, 1>, grid_for(total), 256, 0, stream, a);
}

extern "C" int b200_interpolate(const void* x, int32_t x_dtype, const int64_t* x_strides, void* y, int32_t y_dtype,
                                const int64_t* y_strides, int32_t N, int32_t C, int32_t D, int32_t H, int32_t W,
                                int32_t OD, int32_t OH, int32_t OW, int32_t dims, int32_t mode, float ratio_d,
                                float ratio_h, float ratio_w, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && x_strides && y_strides, "interpolate: null pointer");
  B200_CHECK_ARG(x_dtype >= B200_DT_H16 && x_dtype <= B200_DT_BF16 && (y_dtype == B200_DT_H16 || y_dtype == B200_DT_F32),
                 "interpolate: unknown dtype %d / %d", x_dtype, y_dtype);
  const bool dims_ok = (mode == B200_INTERPOLATE_NEAREST || mode == B200_INTERPOLATE_AREA) ? (dims >= 1 && dims <= 3)
                       : mode == B200_INTERPOLATE_LINEAR                                 ? dims == 1
                       : (mode == B200_INTERPOLATE_BILINEAR || mode == B200_INTERPOLATE_BICUBIC) ? dims == 2
                       : mode == B200_INTERPOLATE_TRILINEAR                              ? dims == 3
                                                                                         : false;
  B200_CHECK_ARG(dims_ok, "interpolate: mode %d does not take %d spatial dims", mode, dims);
  constexpr int kMaxExtent = 1 << 24;  // coordinates are exact in fp32 below this
  B200_CHECK_ARG(N >= 1 && C >= 1 && D >= 1 && H >= 1 && W >= 1 && OD >= 1 && OH >= 1 && OW >= 1 && D <= kMaxExtent &&
                 H <= kMaxExtent && W <= kMaxExtent && OD <= kMaxExtent && OH <= kMaxExtent && OW <= kMaxExtent,
                 "interpolate: bad extents %d x %d x %d x %d x %d -> %d x %d x %d", N, C, D, H, W, OD, OH, OW);
  B200_CHECK_ARG((dims == 3 || (D == 1 && OD == 1)) && (dims >= 2 || (H == 1 && OH == 1)),
                 "interpolate: an axis outside the %d resampled ones must have extent 1", dims);
  for (int i = 0; i < 5; ++i) B200_CHECK_ARG(x_strides[i] >= 0 && y_strides[i] >= 0, "interpolate: negative stride");
  if (mode == B200_INTERPOLATE_AREA) {
    const long long lim = 1ll << 32;
    B200_CHECK_ARG((long long)D * OD + OD <= lim && (long long)H * OH + OH <= lim && (long long)W * OW + OW <= lim,
                   "interpolate: area window arithmetic needs in * out + out <= 2^32 per axis");
  } else {
    const float r[3] = {ratio_d, ratio_h, ratio_w};
    for (int i = 3 - dims; i < 3; ++i)
      B200_CHECK_ARG(r[i] > 0.f && r[i] <= 3.0e38f, "interpolate: ratio %g of axis %d must be positive and finite",
                     (double)r[i], i);
  }
  b200::InterpArgs a;
  a.x = x;
  a.y = y;
  for (int i = 0; i < 5; ++i) {
    a.xs[i] = x_strides[i];
    a.ys[i] = y_strides[i];
  }
  a.x_dt = x_dtype;
  a.y_dt = y_dtype;
  a.N = N; a.C = C; a.D = D; a.H = H; a.W = W; a.OD = OD; a.OH = OH; a.OW = OW; a.dims = dims;
  a.rd = dims == 3 ? ratio_d : 1.f;
  a.rh = dims >= 2 ? ratio_h : 1.f;
  a.rw = ratio_w;
  // 16-byte vectors across channels: an h16 or fp32 input, channel stride 1 and every other stride a multiple of 8
  // elements on both sides, 16-byte aligned pointers, and a voxel stride that leaves room for round_up(C, 8) channels
  const long long c8 = (C + 7) / 8 * 8;
  bool vec = x_dtype <= B200_DT_F32 && x_strides[1] == 1 && y_strides[1] == 1 && (uintptr_t)x % 16 == 0 &&
             (uintptr_t)y % 16 == 0 && x_strides[4] >= c8 && y_strides[4] >= c8;
  for (int i : {0, 2, 3, 4}) vec = vec && x_strides[i] % 8 == 0 && y_strides[i] % 8 == 0;
  cudaError_t e;
  switch (mode) {
    case B200_INTERPOLATE_NEAREST: e = launch_interpolate<INTERP_FAM_NEAREST>(a, vec, stream); break;
    case B200_INTERPOLATE_BICUBIC: e = launch_interpolate<INTERP_FAM_CUBIC>(a, vec, stream); break;
    case B200_INTERPOLATE_AREA: e = launch_interpolate<INTERP_FAM_AREA>(a, vec, stream); break;
    default: e = launch_interpolate<INTERP_FAM_LINEAR>(a, vec, stream); break;
  }
  B200_CUDA(e);
  B200_LAUNCH_CHECK("interpolate_kernel");
  return B200_OK;
}

extern "C" int b200_axpy_h16(const void* a, const void* b, float alpha, void* y, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(a && b && y && n >= 0 && n % 8 == 0, "axpy_h16: element count must be a multiple of 8");
  B200_CHECK_ARG(((uintptr_t)a | (uintptr_t)b | (uintptr_t)y) % 16 == 0, "axpy_h16: pointers must be 16-byte aligned");
  if (n == 0) return B200_OK;
  B200_CUDA(b200::launch_kernel(axpy_h16_kernel, grid_for(n / 8), 256, 0, stream, reinterpret_cast<const uint4*>(a), reinterpret_cast<const uint4*>(b),
                                                       alpha, reinterpret_cast<uint4*>(y), n / 8));
  B200_LAUNCH_CHECK("axpy_h16_kernel");
  return B200_OK;
}


static bool tap_geom_ok(const b200::TapGeom& g) {
  return g.N >= 1 && g.D >= 1 && g.H >= 1 && g.W >= 1 && g.OD >= 1 && g.OH >= 1 && g.OW >= 1 && g.kd >= 1 &&
         g.kh >= 1 && g.kw >= 1 && g.sd >= 1 && g.sh >= 1 && g.sw >= 1 && g.pd >= 0 && g.ph >= 0 && g.pw >= 0;
}

extern "C" int b200_tap_gather(const void* x, int32_t C, int32_t x_pitch, const int32_t* geom, void* out,
                               int32_t out_pitch, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && out && geom && C >= 1 && x_pitch >= C, "tap_gather: bad arguments");
  b200::TapGeom g;
  memcpy(&g, geom, sizeof(g));
  B200_CHECK_ARG(tap_geom_ok(g) && out_pitch >= g.kd * g.kh * g.kw * C && out_pitch % 8 == 0 &&
                 ((uintptr_t)out % 16) == 0, "tap_gather: bad geometry (out_pitch must be a multiple of 8)");
  const long long total = (long long)g.N * g.OD * g.OH * g.OW * (out_pitch / 8);
  B200_CUDA(b200::launch_kernel(tap_gather_kernel, grid_for(total), 256, 0, stream, reinterpret_cast<const h16*>(x), C, x_pitch, g,
                                                        reinterpret_cast<h16*>(out), out_pitch));
  B200_LAUNCH_CHECK("tap_gather_kernel");
  return B200_OK;
}

extern "C" int b200_tap_sum(const float* y, int32_t y_pitch, const int32_t* geom, int32_t cout, const float* bias,
                            void* out, int32_t out_pitch, int32_t out_dtype, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(y && out && geom && cout >= 1 && cout <= 4 && out_pitch >= cout, "tap_sum: 1 <= cout <= 4");
  b200::TapGeom g;
  memcpy(&g, geom, sizeof(g));
  B200_CHECK_ARG(tap_geom_ok(g) && g.sd == 1 && g.sh == 1 && g.sw == 1 && y_pitch >= g.kd * g.kh * g.kw * cout,
                 "tap_sum: bad geometry (stride must be 1)");
  const long long total = (long long)g.N * g.OD * g.OH * g.OW;
  const unsigned grid = grid_for(total);
  switch (cout) {
    case 1: B200_CUDA(b200::launch_kernel(tap_sum_kernel<1>, grid, 256, 0, stream, y, y_pitch, g, bias, out, out_pitch, out_dtype)); break;
    case 2: B200_CUDA(b200::launch_kernel(tap_sum_kernel<2>, grid, 256, 0, stream, y, y_pitch, g, bias, out, out_pitch, out_dtype)); break;
    case 3: B200_CUDA(b200::launch_kernel(tap_sum_kernel<3>, grid, 256, 0, stream, y, y_pitch, g, bias, out, out_pitch, out_dtype)); break;
    default: B200_CUDA(b200::launch_kernel(tap_sum_kernel<4>, grid, 256, 0, stream, y, y_pitch, g, bias, out, out_pitch, out_dtype)); break;
  }
  B200_LAUNCH_CHECK("tap_sum_kernel");
  return B200_OK;
}


// rows of T new tokens per sequence appended to a [B, L, pitch] key/value cache at the device-side position
__global__ void cache_append_kernel(const h16* __restrict__ src, h16* __restrict__ cache, int B,
                                    int T, int L, int pitch, const int* __restrict__ pos_dev) {
  const int pos = *pos_dev;
  const long long total = (long long)B * T * pitch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % pitch);
    const long long r = i / pitch;
    const int t = (int)(r % T), b = (int)(r / T);
    if ((unsigned)(pos + t) < (unsigned)L) cache[((long long)b * L + pos + t) * pitch + c] = src[i];  // 0 <= pos + t < L
  }
}
__global__ void advance_i32_kernel(int* p, int delta) { *p += delta; }

extern "C" int b200_cache_append(const void* src, void* cache, int32_t B, int32_t T, int32_t L, int32_t pitch,
                                 const int32_t* pos_dev, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(src && cache && pos_dev && B >= 1 && T >= 1 && L >= T && pitch >= 1, "cache_append: bad arguments");
  B200_CUDA(b200::launch_kernel(cache_append_kernel, grid_for((long long)B * T * pitch), 256, 0, stream, 
      reinterpret_cast<const h16*>(src), reinterpret_cast<h16*>(cache), B, T, L, pitch, pos_dev));
  B200_LAUNCH_CHECK("cache_append_kernel");
  return B200_OK;
}

extern "C" int b200_advance_i32(int32_t* p, int32_t delta, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p != nullptr, "advance_i32: null pointer");
  B200_CUDA(b200::launch_kernel(advance_i32_kernel, 1, 1, 0, stream, p, delta));
  B200_LAUNCH_CHECK("advance_i32_kernel");
  return B200_OK;
}

extern "C" int b200_embed_tokens(const int64_t* tokens, int64_t M, int32_t seq_len, int32_t pos0, const float* tok_emb,
                                 const float* pos_emb, int32_t C, void* out, int32_t pitch, const int32_t* pos_dev,
                                 void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(tokens && tok_emb && pos_emb && out && M >= 1 && seq_len >= 1 && pos0 >= 0 && C >= 1 && pitch >= C,
                 "embed_tokens: bad arguments");
  B200_CUDA(b200::launch_kernel(embed_tokens_kernel, grid_for(M * pitch), 256, 0, stream, reinterpret_cast<const long long*>(tokens), M, seq_len,
                                                              pos0, tok_emb, pos_emb, C,
                                                              reinterpret_cast<h16*>(out), pitch, pos_dev));
  B200_LAUNCH_CHECK("embed_tokens_kernel");
  return B200_OK;
}

extern "C" int b200_copy_channels(const void* src, int32_t C, int32_t src_pitch, void* dst, int32_t dst_pitch,
                                  int32_t dst_off, int64_t rows, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(src && dst && C >= 1 && src_pitch >= C && dst_pitch >= dst_off + C && rows >= 1, "copy_channels: bad arguments");
  const int vec = (C % 8 == 0 && src_pitch % 8 == 0 && dst_pitch % 8 == 0 && dst_off % 8 == 0 &&
                   ((uintptr_t)src % 16 == 0) && ((uintptr_t)dst % 16 == 0)) ? 8 : 1;
  B200_CUDA(b200::launch_kernel(copy_channels_kernel, grid_for(rows * (C / vec)), 256, 0, stream, reinterpret_cast<const h16*>(src), C, src_pitch,
                                                                     reinterpret_cast<h16*>(dst), dst_pitch, dst_off, rows, vec));
  B200_LAUNCH_CHECK("copy_channels_kernel");
  return B200_OK;
}

extern "C" int b200_geglu(const void* x, int64_t M, int32_t H, int32_t x_pitch, void* y, int32_t y_pitch,
                          void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && M >= 1 && H >= 8 && H % 8 == 0 && x_pitch % 8 == 0 && y_pitch % 8 == 0 &&
                 x_pitch >= 2 * H && y_pitch >= H && ((uintptr_t)x | (uintptr_t)y) % 16 == 0, "geglu: bad arguments");
  B200_CUDA(b200::launch_kernel(geglu_kernel, grid_for(M * (H / 8)), 256, 0, stream, reinterpret_cast<const h16*>(x), M, H, x_pitch,
                                                         reinterpret_cast<h16*>(y), y_pitch));
  B200_LAUNCH_CHECK("geglu_kernel");
  return B200_OK;
}

extern "C" int b200_softmax_rows_partials(const float* s, int64_t M, int32_t S, int64_t s_pitch, const float* partials,
                                          int32_t n_tiles, void* p, int64_t p_pitch, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(s && p && partials && M >= 1 && M < (1ll << 31) && S >= 1 && s_pitch >= S && p_pitch >= S && n_tiles >= 1,
                 "softmax_rows_partials: bad arguments");
  B200_CUDA(b200::launch_kernel(softmax_rows_partials_kernel, (unsigned)M, 256, 0, stream, s, S, s_pitch, reinterpret_cast<const float2*>(partials),
                                                               n_tiles, reinterpret_cast<h16*>(p), p_pitch));
  B200_LAUNCH_CHECK("softmax_rows_partials_kernel");
  return B200_OK;
}

extern "C" int b200_timestep_embedding(const float* t, int32_t N, int32_t dim, float max_period, float* emb,
                                       void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(t && emb && N >= 1 && dim >= 1, "timestep_embedding: bad arguments");
  B200_CHECK_ARG((long long)N * dim < (1ll << 31), "timestep_embedding: N * dim must be below 2^31");
  B200_CUDA(b200::launch_kernel(timestep_embedding_kernel, (N * dim + 255) / 256, 256, 0, stream, t, N, dim, max_period, emb));
  B200_LAUNCH_CHECK("timestep_embedding_kernel");
  return B200_OK;
}

extern "C" int b200_small_linear(const float* x, int32_t M, int32_t K, const float* W, const float* b, int32_t O,
                                 int32_t act_in, int32_t act_out, float* y, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && W && y && M >= 1 && M <= 4096 && K >= 1 && O >= 1, "small_linear: bad arguments");
  const bool vec = (K % 128 == 0) && (((uintptr_t)x | (uintptr_t)W) & 15) == 0;
  if (vec) B200_CUDA(b200::launch_kernel(small_linear_kernel<true>, (O + 7) / 8, 256, 0, stream, x, M, K, W, b, O, act_in, act_out, y));
  else B200_CUDA(b200::launch_kernel(small_linear_kernel<false>, (O + 7) / 8, 256, 0, stream, x, M, K, W, b, O, act_in, act_out, y));
  B200_LAUNCH_CHECK("small_linear_kernel");
  return B200_OK;
}

extern "C" int b200_ddim_step(const float* model_out, const float* sample, const float* noise, const b200_ddim_coef* c,
                              float* prev_sample, float* pred_x0, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(model_out && sample && c && prev_sample && n >= 1, "ddim_step: bad arguments");
  const bool vec = (((uintptr_t)model_out | (uintptr_t)sample | (uintptr_t)noise | (uintptr_t)prev_sample | (uintptr_t)pred_x0) & 15) == 0;
  if (vec) B200_CUDA(b200::launch_kernel(ddim_step_kernel<1>, grid_for((n + 7) / 8, 256, 16), 256, 0, stream, model_out, sample, noise, *c, prev_sample, pred_x0, (long long)n));
  else B200_CUDA(b200::launch_kernel(ddim_step_kernel<0>, grid_for(n), 256, 0, stream, model_out, sample, noise, *c, prev_sample, pred_x0, (long long)n));
  B200_LAUNCH_CHECK("ddim_step_kernel");
  return B200_OK;
}

extern "C" int b200_ddpm_step(const float* model_out, const float* sample, const float* noise, const float* pred_var,
                              const b200_ddpm_coef* c, float* prev_sample, float* pred_x0, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(model_out && sample && c && prev_sample && n >= 1, "ddpm_step: bad arguments");
  B200_CHECK_ARG(c->var_mode == 0 || pred_var, "ddpm_step: learned variance needs pred_var");
  B200_CUDA(b200::launch_kernel(ddpm_step_kernel, grid_for(n), 256, 0, stream, model_out, sample, noise, pred_var, *c, prev_sample, pred_x0, n));
  B200_LAUNCH_CHECK("ddpm_step_kernel");
  return B200_OK;
}

extern "C" int b200_pndm_step(const float* const* hist, const float* sample, const b200_pndm_coef* c, float* prev_sample,
                              float* eps_out, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(hist && c && c->n_hist >= 1 && c->n_hist <= 4 && n >= 1, "pndm_step: bad arguments");
  B200_CHECK_ARG(prev_sample == nullptr || sample != nullptr, "pndm_step: prev_sample needs sample");
  PndmPtrs hp;
  for (int k = 0; k < 4; ++k) hp.h[k] = k < c->n_hist ? hist[k] : nullptr;
  for (int k = 0; k < c->n_hist; ++k) B200_CHECK_ARG(hp.h[k], "pndm_step: null history tensor %d", k);
  B200_CUDA(b200::launch_kernel(pndm_step_kernel, grid_for(n), 256, 0, stream, hp, sample, *c, prev_sample, eps_out, n));
  B200_LAUNCH_CHECK("pndm_step_kernel");
  return B200_OK;
}

extern "C" int b200_add_noise(const float* x0, const float* noise, const float* ca, const float* cb, float sign_b,
                              int32_t N, int64_t per_sample, float* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x0 && noise && ca && cb && out && N >= 1 && N <= 65535 && per_sample >= 1, "add_noise: bad arguments");
  dim3 grid(grid_for(per_sample, 256, 4), N);
  B200_CUDA(b200::launch_kernel(add_noise_kernel, grid, 256, 0, stream, x0, noise, ca, cb, sign_b, per_sample, out));
  B200_LAUNCH_CHECK("add_noise_kernel");
  return B200_OK;
}

extern "C" int b200_exp_half_clamped(const float* log_var, float lo, float hi, float* sigma, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(log_var && sigma && n >= 1, "exp_half_clamped: bad arguments");
  B200_CUDA(b200::launch_kernel(exp_half_clamped_kernel, grid_for(n), 256, 0, stream, log_var, lo, hi, sigma, n));
  B200_LAUNCH_CHECK("exp_half_clamped_kernel");
  return B200_OK;
}

extern "C" int b200_fma_f32(const float* a, const float* b, const float* c, float* out, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(a && b && c && out && n >= 1, "fma_f32: bad arguments");
  B200_CUDA(b200::launch_kernel(fma_f32_kernel, grid_for(n), 256, 0, stream, a, b, c, out, n));
  B200_LAUNCH_CHECK("fma_f32_kernel");
  return B200_OK;
}

extern "C" int b200_scale_f32(const float* x, float mul, float div, float* out, int64_t n, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && out && n >= 1 && div != 0.f, "scale_f32: bad arguments");
  B200_CUDA(b200::launch_kernel(scale_f32_kernel, grid_for(n), 256, 0, stream, x, mul, div, out, n));
  B200_LAUNCH_CHECK("scale_f32_kernel");
  return B200_OK;
}

extern "C" int b200_ddpm_kl(const float* x0, const float* xt, const float* model_out, const b200_kl_coef* c, float* kl_out,
                            double* sample_sum, int32_t N, int64_t per_sample, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x0 && xt && model_out && c && sample_sum && N >= 1 && N <= 65535 && per_sample >= 1, "ddpm_kl: bad arguments");
  dim3 grid(grid_for(per_sample, 256, 4), N);
  B200_CUDA(b200::launch_kernel(ddpm_kl_kernel, grid, 256, 0, stream, x0, xt, model_out, *c, kl_out, sample_sum, per_sample));
  B200_LAUNCH_CHECK("ddpm_kl_kernel");
  return B200_OK;
}
