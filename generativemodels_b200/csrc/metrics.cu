// Sample-quality metrics (generative/metrics/{ssim,ms_ssim,mmd}.py of the reference): SSIM / CS partial sums in one
// separable pass per scale, the fp32 2x average pooling between MS-SSIM scales, the per-item finish of SSIM and
// MS-SSIM, and MMD with the linear kernel as one column reduction.  Contracts: include/b200gen_metrics.h.
#include "common.cuh"
#include "../../include/b200gen_metrics.h"

namespace b200 {
namespace {

constexpr int kTW = 32;          // output tile width (one warp across W)
constexpr int kThreads = 256;
constexpr int kMaxSmem = 224 * 1024;  // dynamic; block_sum2 adds 128 static bytes

__device__ __forceinline__ float load_any(const void* p, int dt, int64_t i) {
  switch (dt) {
    case B200_DT_F32: return static_cast<const float*>(p)[i];
    case B200_DT_F64: return static_cast<float>(static_cast<const double*>(p)[i]);
    case B200_DT_FP16: return __half2float(static_cast<const __half*>(p)[i]);
    default: return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
  }
}

// Sum of (a, b) over the block in a fixed order: warp butterflies, then warp 0 over the per-warp sums.
__device__ __forceinline__ double2 block_sum2(double a, double b) {
  __shared__ double2 red[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  __syncthreads();
  if (lane == 0) red[warp] = make_double2(a, b);
  __syncthreads();
  double2 r = make_double2(0.0, 0.0);
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) {
      r.x += red[w].x;
      r.y += red[w].y;
    }
  return r;  // valid in thread 0
}

struct SsimGeom {
  int TH, DC, tiles_w, tiles_h, chunks, OD, OH, OW;
  size_t smem;
};

size_t ssim_smem(int TH, int kd, int kh, int kw) {
  const size_t SR = TH + kh - 1, SW = kTW + kw - 1;
  return sizeof(float) * (2 * SR * SW + 5 * SR * kTW + 5 * (size_t)kd * TH * kTW);
}

// Tile height: the tallest of 8, 4, 2, 1 rows whose staging, W-filtered rows and ring of kd filtered planes fit in
// shared memory.  Depth chunk (3-D): the most output planes per CTA, from 64 down to 8, that still gives the grid four
// CTAs per SM.
bool ssim_geom(const b200_ssim_params* p, SsimGeom* g) {
  g->OD = p->D - p->kd + 1;
  g->OH = p->H - p->kh + 1;
  g->OW = p->W - p->kw + 1;
  g->TH = 0;
  for (int th = 8; th >= 1; th /= 2)
    if (ssim_smem(th, p->kd, p->kh, p->kw) <= (size_t)kMaxSmem) {
      g->TH = th;
      break;
    }
  if (!g->TH) return false;
  g->smem = ssim_smem(g->TH, p->kd, p->kh, p->kw);
  g->tiles_w = (g->OW + kTW - 1) / kTW;
  g->tiles_h = (g->OH + g->TH - 1) / g->TH;
  g->DC = g->OD;
  if (g->OD > 1) {
    const long long want = 4ll * sm_count();
    g->DC = 64;
    while (g->DC > 8 && (long long)g->tiles_w * g->tiles_h * ((g->OD + g->DC - 1) / g->DC) * p->N * p->C < want)
      g->DC /= 2;
    g->DC = g->DC < g->OD ? g->DC : g->OD;
  }
  g->chunks = (g->OD + g->DC - 1) / g->DC;
  return true;
}

// One CTA: item n, channel c, a TH x 32 tile of output rows / columns and DC output planes.  Per input plane: stage x
// and y (fp32), filter x, y, x^2, y^2, xy along W, then along H into slot (z - od0) % kd of a ring of filtered planes;
// once kd planes are in the ring, filter along D and form SSIM and CS per valid voxel.
__global__ void __launch_bounds__(kThreads) ssim_kernel(const b200_ssim_params p, const SsimGeom g) {
  extern __shared__ float sm[];
  const int TH = g.TH, SW = kTW + p.kw - 1, SR = TH + p.kh - 1, tile = TH * kTW;
  float* sx = sm;
  float* sy = sx + SR * SW;
  float* wf = sy + SR * SW;     // [5][SR][32]
  float* ring = wf + 5 * SR * kTW;  // [kd][5][TH][32]
  const int n = blockIdx.z, c = blockIdx.y;
  int t = blockIdx.x;
  const int w0 = (t % g.tiles_w) * kTW;
  t /= g.tiles_w;
  const int h0 = (t % g.tiles_h) * TH;
  const int od0 = (t / g.tiles_h) * g.DC;
  const int od1 = min(od0 + g.DC, g.OD);
  const int64_t xb = n * p.x_strides[0] + c * p.x_strides[1], yb = n * p.y_strides[0] + c * p.y_strides[1];
  const int tid = threadIdx.x;
  double acc_s = 0.0, acc_c = 0.0;

  for (int z = od0; z < od1 + p.kd - 1; ++z) {
    for (int i = tid; i < SR * SW; i += kThreads) {
      const int hh = h0 + i / SW, ww = w0 + i % SW;
      float a = 0.f, b = 0.f;
      if (hh < p.H && ww < p.W) {
        a = load_any(p.x, p.x_dtype, xb + z * p.x_strides[2] + hh * p.x_strides[3] + ww * p.x_strides[4]);
        b = load_any(p.y, p.y_dtype, yb + z * p.y_strides[2] + hh * p.y_strides[3] + ww * p.y_strides[4]);
      }
      sx[i] = a;
      sy[i] = b;
    }
    __syncthreads();
    for (int i = tid; i < SR * kTW; i += kThreads) {
      const float* px = sx + (i / kTW) * SW + i % kTW;
      const float* py = sy + (i / kTW) * SW + i % kTW;
      float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
      for (int q = 0; q < p.kw; ++q) {
        const float wt = p.taps_w[q], a = px[q], b = py[q];
        m0 = fmaf(wt, a, m0);
        m1 = fmaf(wt, b, m1);
        m2 = fmaf(wt, a * a, m2);
        m3 = fmaf(wt, b * b, m3);
        m4 = fmaf(wt, a * b, m4);
      }
      const int plane = SR * kTW;
      wf[i] = m0;
      wf[plane + i] = m1;
      wf[2 * plane + i] = m2;
      wf[3 * plane + i] = m3;
      wf[4 * plane + i] = m4;
    }
    __syncthreads();
    float* slot = ring + ((z - od0) % p.kd) * 5 * tile;
    for (int i = tid; i < tile; i += kThreads) {
      const int plane = SR * kTW;
      const float* src = wf + i;  // row i / 32 of the tile, column i % 32
      float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
      for (int q = 0; q < p.kh; ++q) {
        const float wt = p.taps_h[q];
#pragma unroll
        for (int k = 0; k < 5; ++k) m[k] = fmaf(wt, src[k * plane + q * kTW], m[k]);
      }
#pragma unroll
      for (int k = 0; k < 5; ++k) slot[k * tile + i] = m[k];
    }
    __syncthreads();
    if (z >= od0 + p.kd - 1) {
      const int o = z - p.kd + 1;
      for (int i = tid; i < tile; i += kThreads) {
        const int oh = h0 + i / kTW, ow = w0 + i % kTW;
        if (oh >= g.OH || ow >= g.OW) continue;
        float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        for (int q = 0; q < p.kd; ++q) {
          const float wt = p.taps_d[q];
          const float* s = ring + ((o + q - od0) % p.kd) * 5 * tile + i;
#pragma unroll
          for (int k = 0; k < 5; ++k) m[k] = fmaf(wt, s[k * tile], m[k]);
        }
        const float mx = m[0] * p.scale, my = m[1] * p.scale, mxx = m[2] * p.scale, myy = m[3] * p.scale,
                    mxy = m[4] * p.scale;
        const float sgx = mxx - mx * mx, sgy = myy - my * my, sgxy = mxy - mx * my;
        const float cs = (2.f * sgxy + p.c2) / (sgx + sgy + p.c2);
        const float ss = ((2.f * mx * my + p.c1) / (mx * mx + my * my + p.c1)) * cs;
        acc_s += ss;
        acc_c += cs;
        if (p.ssim_map || p.cs_map) {
          const int64_t at = (((int64_t)(n * p.C + c) * g.OD + o) * g.OH + oh) * g.OW + ow;
          if (p.ssim_map) p.ssim_map[at] = ss;
          if (p.cs_map) p.cs_map[at] = cs;
        }
      }
    }
  }
  const double2 r = block_sum2(acc_s, acc_c);
  if (tid == 0) {
    double* dst = p.partials + 2 * ((int64_t)n * p.C * gridDim.x + (int64_t)c * gridDim.x + blockIdx.x);
    dst[0] = r.x;
    dst[1] = r.y;
  }
}

__global__ void __launch_bounds__(kThreads) ssim_combine_kernel(const b200_ssim_combine_params p) {
  const int n = blockIdx.x;
  float ms = 1.f;
  for (int s = 0; s < p.n_scales; ++s) {
    const double* part = p.partials[s] + 2 * (int64_t)n * p.slots[s];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < p.slots[s]; i += kThreads) {
      a += part[2 * i];
      b += part[2 * i + 1];
    }
    const double2 r = block_sum2(a, b);
    if (threadIdx.x == 0) {
      const float ssim = static_cast<float>(r.x / (double)p.count[s]);
      const float cs = static_cast<float>(r.y / (double)p.count[s]);
      if (p.ssim_mean) p.ssim_mean[s * p.N + n] = ssim;
      if (p.cs_mean) p.cs_mean[s * p.N + n] = cs;
      const float v = s == p.n_scales - 1 ? ssim : cs;
      ms *= powf(fmaxf(v, 0.f), p.weights[s]);
    }
  }
  if (threadIdx.x == 0 && p.ms_ssim) p.ms_ssim[n] = ms;
}

__global__ void avgpool2_f32_kernel(const void* x, int dt, int64_t s0, int64_t s1, int64_t s2, int64_t s3, int64_t s4, int N, int C, int OD, int OH, int OW, int pd,
                                    float* y) {
  const int64_t total = (int64_t)N * C * OD * OH * OW;
  const float div = pd == 2 ? 8.f : 4.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    const int ow = t % OW;
    t /= OW;
    const int oh = t % OH;
    t /= OH;
    const int od = t % OD;
    t /= OD;
    const int c = t % C;
    const int n = t / C;
    const int64_t base = n * s0 + c * s1 + (int64_t)od * pd * s2 + (int64_t)oh * 2 * s3 + (int64_t)ow * 2 * s4;
    float sum = 0.f;
    for (int dd = 0; dd < pd; ++dd)
      for (int hh = 0; hh < 2; ++hh)
        for (int ww = 0; ww < 2; ++ww) sum += load_any(x, dt, base + dd * s2 + hh * s3 + ww * s4);
    y[i] = sum / div;
  }
}

struct MmdArgs {
  const void* y;
  const void* p;
  int y_dt, p_dt;
  int64_t ys[5], ps[5], shape[5];
  int64_t V;
};

template <bool kDense>
__global__ void __launch_bounds__(kThreads) mmd_partial_kernel(const MmdArgs a, double* part) {
  double acc = 0.0;
  for (int64_t v = blockIdx.x * (int64_t)kThreads + threadIdx.x; v < a.V; v += (int64_t)gridDim.x * kThreads) {
    int64_t oy = v, op = v;
    if (!kDense) {
      int64_t t = v;
      const int64_t i4 = t % a.shape[4];
      t /= a.shape[4];
      const int64_t i3 = t % a.shape[3];
      t /= a.shape[3];
      const int64_t i2 = t % a.shape[2];
      const int64_t i1 = t / a.shape[2];
      oy = i1 * a.ys[1] + i2 * a.ys[2] + i3 * a.ys[3] + i4 * a.ys[4];
      op = i1 * a.ps[1] + i2 * a.ps[2] + i3 * a.ps[3] + i4 * a.ps[4];
    }
    double d = 0.0;
    for (int64_t b = 0; b < a.shape[0]; ++b)
      d += (double)load_any(a.y, a.y_dt, b * a.ys[0] + oy) - (double)load_any(a.p, a.p_dt, b * a.ps[0] + op);
    acc = fma(d, d, acc);
  }
  const double2 r = block_sum2(acc, 0.0);
  if (threadIdx.x == 0) part[blockIdx.x] = r.x;
}

__global__ void __launch_bounds__(kThreads) mmd_finish_kernel(const double* part, int n_part, double denom, float* out) {
  double a = 0.0;
  for (int i = threadIdx.x; i < n_part; i += kThreads) a += part[i];
  const double2 r = block_sum2(a, 0.0);
  if (threadIdx.x == 0) *out = static_cast<float>(r.x / denom);
}

int mmd_blocks(int64_t V) {
  const int64_t b = (V + 4 * kThreads - 1) / (4 * kThreads);
  return (int)(b < 1024 ? (b < 1 ? 1 : b) : 1024);
}

bool metric_dtype_ok(int dt) {
  return dt == B200_DT_F32 || dt == B200_DT_F64 || dt == B200_DT_FP16 || dt == B200_DT_BF16;
}

}  // namespace
}  // namespace b200

using b200::SsimGeom;

extern "C" int64_t b200_ssim_workspace_bytes(const b200_ssim_params* p) {
  SsimGeom g;
  if (!p || p->N < 1 || p->C < 1 || p->kd < 1 || p->kh < 1 || p->kw < 1 || p->kd > p->D || p->kh > p->H ||
      p->kw > p->W || !b200::ssim_geom(p, &g))
    return -1;
  return (int64_t)p->N * p->C * g.tiles_w * g.tiles_h * g.chunks * 2 * (int64_t)sizeof(double);
}

extern "C" int b200_ssim(const b200_ssim_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->x && p->y && p->partials, "ssim: null pointer");
  B200_CHECK_ARG(b200::metric_dtype_ok(p->x_dtype) && b200::metric_dtype_ok(p->y_dtype), "ssim: unknown dtype %d / %d",
                 p->x_dtype, p->y_dtype);
  B200_CHECK_ARG(p->N >= 1 && p->C >= 1 && p->D >= 1 && p->H >= 1 && p->W >= 1 && p->N <= 65535 && p->C <= 65535,
                 "ssim: bad extents %d x %d x %d x %d x %d", p->N, p->C, p->D, p->H, p->W);
  B200_CHECK_ARG(p->kd >= 1 && p->kh >= 1 && p->kw >= 1 && p->kd <= B200_SSIM_MAX_K && p->kh <= B200_SSIM_MAX_K &&
                     p->kw <= B200_SSIM_MAX_K,
                 "ssim: kernel %d x %d x %d outside 1..%d", p->kd, p->kh, p->kw, B200_SSIM_MAX_K);
  B200_CHECK_ARG(p->kd <= p->D && p->kh <= p->H && p->kw <= p->W, "ssim: kernel %d x %d x %d larger than %d x %d x %d",
                 p->kd, p->kh, p->kw, p->D, p->H, p->W);
  for (int i = 0; i < 5; ++i)
    B200_CHECK_ARG(p->x_strides[i] >= 0 && p->y_strides[i] >= 0, "ssim: negative stride");
  SsimGeom g;
  if (!b200::ssim_geom(p, &g)) {
    b200::set_error("ssim: a %d x %d x %d kernel does not fit one tile in shared memory", p->kd, p->kh, p->kw);
    return B200_ENOTSUP;
  }
  B200_CUDA(cudaFuncSetAttribute(b200::ssim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, b200::kMaxSmem));
  const dim3 grid(g.tiles_w * g.tiles_h * g.chunks, p->C, p->N);
  B200_CUDA(b200::launch_kernel(b200::ssim_kernel, grid, dim3(b200::kThreads), g.smem, stream, *p, g));
  B200_LAUNCH_CHECK("ssim_kernel");
  return B200_OK;
}

extern "C" int b200_ssim_combine(const b200_ssim_combine_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->N >= 1 && p->n_scales >= 1 && p->n_scales <= B200_SSIM_MAX_SCALES,
                 "ssim_combine: bad N / scale count");
  for (int s = 0; s < p->n_scales; ++s)
    B200_CHECK_ARG(p->partials[s] && p->slots[s] >= 1 && p->count[s] >= 1, "ssim_combine: scale %d has no partials", s);
  B200_CUDA(b200::launch_kernel(b200::ssim_combine_kernel, dim3(p->N), dim3(b200::kThreads), 0, stream, *p));
  B200_LAUNCH_CHECK("ssim_combine_kernel");
  return B200_OK;
}

extern "C" int b200_avgpool2_f32(const void* x, int32_t x_dtype, const int64_t* x_strides, int32_t N, int32_t C,
                                 int32_t D, int32_t H, int32_t W, int32_t dims, float* y, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && x_strides, "avgpool2_f32: null pointer");
  B200_CHECK_ARG(b200::metric_dtype_ok(x_dtype), "avgpool2_f32: unknown dtype %d", x_dtype);
  B200_CHECK_ARG(dims == 2 || dims == 3, "avgpool2_f32: dims must be 2 or 3, got %d", dims);
  B200_CHECK_ARG(dims == 3 || D == 1, "avgpool2_f32: a 2-D pooling needs D == 1");
  const int OD = dims == 3 ? D / 2 : 1, OH = H / 2, OW = W / 2;
  B200_CHECK_ARG(N >= 1 && C >= 1 && OD >= 1 && OH >= 1 && OW >= 1, "avgpool2_f32: output would be empty");
  const int64_t total = (int64_t)N * C * OD * OH * OW;
  const int blocks = (int)((total + 255) / 256 < 65536 ? (total + 255) / 256 : 65536);
  B200_CUDA(b200::launch_kernel(b200::avgpool2_f32_kernel, dim3(blocks), dim3(256), 0, stream, x, x_dtype,
                                x_strides[0], x_strides[1], x_strides[2], x_strides[3], x_strides[4], N, C, OD, OH, OW,
                                dims == 3 ? 2 : 1, y));
  B200_LAUNCH_CHECK("avgpool2_f32_kernel");
  return B200_OK;
}

extern "C" int64_t b200_mmd_workspace_bytes(const int64_t* shape) {
  if (!shape) return -1;
  return (int64_t)b200::mmd_blocks(shape[1] * shape[2] * shape[3] * shape[4]) * (int64_t)sizeof(double);
}

extern "C" int b200_mmd(const void* y, int32_t y_dtype, const int64_t* y_strides, const void* y_pred,
                        int32_t y_pred_dtype, const int64_t* y_pred_strides, const int64_t* shape, double* workspace,
                        float* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(y && y_pred && y_strides && y_pred_strides && shape && workspace && out, "mmd: null pointer");
  B200_CHECK_ARG(b200::metric_dtype_ok(y_dtype) && b200::metric_dtype_ok(y_pred_dtype), "mmd: unknown dtype %d / %d",
                 y_dtype, y_pred_dtype);
  b200::MmdArgs a;
  a.y = y;
  a.p = y_pred;
  a.y_dt = y_dtype;
  a.p_dt = y_pred_dtype;
  bool dense = true;
  int64_t inner = 1;
  for (int i = 4; i >= 0; --i) {
    B200_CHECK_ARG(shape[i] >= 1 && y_strides[i] >= 0 && y_pred_strides[i] >= 0, "mmd: bad extent or stride on axis %d",
                   i);
    a.shape[i] = shape[i];
    a.ys[i] = y_strides[i];
    a.ps[i] = y_pred_strides[i];
    if (i >= 1) {
      dense = dense && (shape[i] == 1 || (y_strides[i] == inner && y_pred_strides[i] == inner));
      inner *= shape[i];
    }
  }
  a.V = inner;
  const int blocks = b200::mmd_blocks(a.V);
  if (dense)
    B200_CUDA(b200::launch_kernel(b200::mmd_partial_kernel<true>, dim3(blocks), dim3(b200::kThreads), 0, stream, a,
                                  workspace));
  else
    B200_CUDA(b200::launch_kernel(b200::mmd_partial_kernel<false>, dim3(blocks), dim3(b200::kThreads), 0, stream, a,
                                  workspace));
  B200_LAUNCH_CHECK("mmd_partial_kernel");
  const double denom = (double)shape[0] * (double)shape[0] * (double)a.V;
  B200_CUDA(b200::launch_kernel(b200::mmd_finish_kernel, dim3(1), dim3(b200::kThreads), 0, stream,
                                (const double*)workspace, blocks, denom, out));
  B200_LAUNCH_CHECK("mmd_finish_kernel");
  return B200_OK;
}
