// GroupNorm (+SiLU) and LayerNorm on channels-last bf16 (HBM-bound; 128-bit coalesced accesses).
//
// Reference arithmetic: nn.GroupNorm(num_groups, C, eps, affine=True) followed by nn.SiLU in
// ResnetBlock.forward (diffusion_model_unet.py:669-696), AttentionBlock (372, 418-422), the output head
// (1853-1855) and the AutoencoderKL ResBlock/AttentionBlock (autoencoderkl.py:139-146, 229); nn.LayerNorm in
// BasicTransformerBlock (diffusion_model_unet.py:221-223).
//
// GroupNorm is split in two phases so that neither pass re-reads more than it must:
//   stats : every block reduces a slab of voxels to per-channel (sum, sumsq) partials of x - p in fp32, where the
//           pivot p is one element of the group (its first channel at voxel 0); a tiny finalize kernel folds the
//           partials -> group mean / rstd in fp64 and emits the per-(n, c) affine pair a = rstd * gamma,
//           b = beta - mean * a.  Summing x - p instead of x keeps E[x^2] - mean^2 from cancelling when a group's
//           mean is large against its spread (the fp32 error of a raw sum of squares grows with (mean / std)^2).
//   apply : y = silu(a * x + b), one read + one write, optionally reading a virtual concat of two tensors
//           (the up-path torch.cat at diffusion_model_unet.py:1232/1340/1461 is never materialised raw).
#include "common.cuh"

namespace b200 {

static constexpr int kGnMaxChunks = 512;

// The statistics pivot of the group whose first channel is c (of the virtual concat): x[n, voxel 0, c].
__device__ __forceinline__ float gn_pivot(const h16* x0, const h16* x1, int C0, int pitch0, int pitch1,
                                          long long spatial, int n, int c) {
  return c < C0 ? h2f(x0[(long long)n * spatial * pitch0 + c]) : h2f(x1[(long long)n * spatial * pitch1 + (c - C0)]);
}

// ---- stats --------------------------------------------------------------------------------------
// grid = (chunks, N); block = CV * rows threads, CV = C_total / VEC channel vectors.
template <int VEC>
__global__ void gn_partial_kernel(const h16* __restrict__ x0, const h16* __restrict__ x1,
                                  int C0, int C1, int pitch0, int pitch1, long long spatial, int cpg,
                                  long long vox_per_chunk, float* __restrict__ partial) {
  const int C = C0 + C1;
  const int CV = C / VEC;
  const int rows = blockDim.x / CV;
  const int cv = threadIdx.x % CV;
  const int row = threadIdx.x / CV;
  const int n = blockIdx.y;
  const int chunk = blockIdx.x;
  const long long s0 = (long long)chunk * vox_per_chunk;
  long long s1 = s0 + vox_per_chunk;
  if (s1 > spatial) s1 = spatial;

  const int c = cv * VEC;
  const h16* src;
  int pitch;
  int cc;
  if (c < C0) { src = x0; pitch = pitch0; cc = c; }
  else        { src = x1; pitch = pitch1; cc = c - C0; }
  src += (long long)n * spatial * pitch + cc;

  float sum[VEC], sq[VEC], piv[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    sum[j] = 0.f;
    sq[j] = 0.f;
    piv[j] = gn_pivot(x0, x1, C0, pitch0, pitch1, spatial, n, (c + j) / cpg * cpg);
  }

  if (row < rows) {
    long long s = s0 + row;
    if constexpr (VEC == 8) {
      // four independent 16-byte loads in flight per thread (a one-read streaming pass: bytes in flight per SM is what
      // sets its bandwidth — one dependent load per iteration left it at 0.70 of the copy bandwidth)
      for (; s + 3ll * rows < s1; s += 4ll * rows) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(src + (s + (long long)u * rows) * pitch));
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float f[8];
          unpack8(v[u], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float d = f[j] - piv[j];
            sum[j] += d;
            sq[j] = fmaf(d, d, sq[j]);
          }
        }
      }
    }
    for (; s < s1; s += rows) {
      float f[VEC];
      if constexpr (VEC == 8) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(src + s * pitch));
        unpack8(v, f);
      } else {
#pragma unroll
        for (int j = 0; j < VEC; ++j) f[j] = h2f(src[s * pitch + j]);
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float d = f[j] - piv[j];
        sum[j] += d;
        sq[j] = fmaf(d, d, sq[j]);
      }
    }
  }
  // reduce the `rows` threads that share a channel vector through shared memory
  extern __shared__ float sm[];   // [rows][C][2]
  if (row < rows) {
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      sm[((long long)row * C + c + j) * 2 + 0] = sum[j];
      sm[((long long)row * C + c + j) * 2 + 1] = sq[j];
    }
  }
  __syncthreads();
  float* out = partial + (((long long)n * gridDim.x + chunk) * C) * 2;
  for (int i = threadIdx.x; i < C * 2; i += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < rows; ++r) acc += sm[(long long)r * C * 2 + i];
    out[i] = acc;
  }
}

// grid = (groups, N); folds the partials of one group in fp64 around the group mean and writes the affine pairs.
__global__ void gn_finalize_kernel(const float* __restrict__ partial, const h16* __restrict__ x0,
                                   const h16* __restrict__ x1, int C0, int pitch0, int pitch1, int chunks, int C,
                                   int groups, long long spatial, float eps, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* __restrict__ affine) {
  const int g = blockIdx.x, n = blockIdx.y;
  const int cpg = C / groups;
  double s = 0.0, q = 0.0;
  // four (sum, sum of squares) pairs in flight per thread: a plain load -> add loop is ~9 dependent L2 round trips per
  // thread for a few kilobytes of partials; same addition order
  const int total = chunks * cpg;
  int i = threadIdx.x;
  for (; i + 3 * (int)blockDim.x < total; i += 4 * blockDim.x) {
    float2 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int ii = i + u * blockDim.x;
      const int ch = ii / cpg, c = g * cpg + ii % cpg;
      v[u] = __ldg(reinterpret_cast<const float2*>(partial + (((long long)n * chunks + ch) * C + c) * 2));
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) { s += (double)v[u].x; q += (double)v[u].y; }
  }
  for (; i < total; i += blockDim.x) {
    const int ch = i / cpg, c = g * cpg + i % cpg;
    const float2 v = __ldg(reinterpret_cast<const float2*>(partial + (((long long)n * chunks + ch) * C + c) * 2));
    s += (double)v.x;
    q += (double)v.y;
  }
  __shared__ double ss[32], sq[32];
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { ss[w] = s; sq[w] = q; }
  __syncthreads();
  if (w == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    s = l < nw ? ss[l] : 0.0;
    q = l < nw ? sq[l] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (l == 0) { ss[0] = s; sq[0] = q; }
  }
  __syncthreads();
  // the partials are sums of x - p: mean = p + E[x - p], var = E[(x - p)^2] - E[x - p]^2
  const double cnt = (double)spatial * cpg;
  const double dm = ss[0] / cnt;
  double var = sq[0] / cnt - dm * dm;
  if (var < 0.0) var = 0.0;
  const double mean = (double)gn_pivot(x0, x1, C0, pitch0, pitch1, spatial, n, g * cpg) + dm;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  for (int j = threadIdx.x; j < cpg; j += blockDim.x) {
    const int c = g * cpg + j;
    const float a = rstd * gamma[c];
    affine[((long long)n * C + c) * 2 + 0] = a;
    affine[((long long)n * C + c) * 2 + 1] = beta[c] - (float)mean * a;
  }
}


// ---- finalize from igemm-epilogue partials ----------------------------------------------------------
// partial_i[n][slot][C_i/8][2]; consumer group g spans cpg channels = cpg/8 producer groups of one source.
__global__ void gn_finalize_partials_kernel(const float* __restrict__ p0, const float* __restrict__ p1, int slots0,
                                            int slots1, int C0, int C1, int sh0, int sh1, int groups, long long spatial,
                                            float eps, const float* __restrict__ gamma, const float* __restrict__ beta,
                                            float* __restrict__ affine) {
  const int g = blockIdx.x, n = blockIdx.y;
  const int C = C0 + C1;
  const int cpg = C / groups;
  const int c_first = g * cpg;
  const float* src;
  int slots, g8_total, g8_first, sh;            // producer groups of 1 << sh channels (8 or 4)
  if (c_first < C0) { src = p0; slots = slots0; sh = sh0; g8_total = C0 >> sh; g8_first = c_first >> sh; }
  else { src = p1; slots = slots1; sh = sh1; g8_total = C1 >> sh; g8_first = (c_first - C0) >> sh; }
  const int sub = cpg >> sh;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < slots * sub; i += blockDim.x) {
    const int slot = i / sub, j = i - slot * sub;
    const float* e = src + (((long long)n * slots + slot) * g8_total + g8_first + j) * 2;
    s += (double)e[0];
    q += (double)e[1];
  }
  __shared__ double ss[32], sq[32];
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { ss[w] = s; sq[w] = q; }
  __syncthreads();
  if (w == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    s = l < nw ? ss[l] : 0.0;
    q = l < nw ? sq[l] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (l == 0) { ss[0] = s; sq[0] = q; }
  }
  __syncthreads();
  const double cnt = (double)spatial * cpg;
  const double mean = ss[0] / cnt;
  double var = sq[0] / cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  for (int j = threadIdx.x; j < cpg; j += blockDim.x) {
    const int c = c_first + j;
    const float a = rstd * gamma[c];
    affine[((long long)n * C + c) * 2 + 0] = a;
    affine[((long long)n * C + c) * 2 + 1] = beta[c] - (float)mean * a;
  }
}

// ---- apply --------------------------------------------------------------------------------------
// grid = (chunks, N); block = CV * rows threads.  A thread owns one 8-channel vector for its whole slab, so its
// affine pairs live in registers and the inner loop is: 128-bit load, 8 FMA, 8 SiLU, 128-bit store (no index
// division, no shared-memory traffic).
__device__ __forceinline__ float silu_fast(float x) {
  // x * sigmoid(x) with ex2.approx + rcp.approx (2 SFU ops, ~2 ulp): the full-precision division of x / (1 + e^-x)
  // costs ~10 ALU instructions per element and made this HBM-bound pass instruction-bound.
  return __fdividef(x, 1.0f + __expf(-x));
}
// the activations the GroupNorm apply passes take: none, SiLU, LeakyReLU(0.01), LeakyReLU(0.2)
__device__ __forceinline__ float gn_act(float t, int act) {
  if (act == B200_ACT_SILU) return silu_fast(t);
  if (act == B200_ACT_LEAKYRELU) return t > 0.0f ? t : 0.01f * t;
  if (act == B200_ACT_LEAKYRELU02) return t > 0.0f ? t : 0.2f * t;
  return t;
}
__host__ __forceinline__ bool gn_act_ok(int act) {
  return act == B200_ACT_NONE || act == B200_ACT_SILU || act == B200_ACT_LEAKYRELU || act == B200_ACT_LEAKYRELU02;
}

template <int VEC>
__global__ void gn_apply_kernel(const h16* __restrict__ x0, const h16* __restrict__ x1,
                                int C0, int C1, int pitch0, int pitch1, long long spatial, long long vox_per_chunk,
                                const float* __restrict__ affine, int act, h16* __restrict__ y,
                                int y_pitch) {
  const int C = C0 + C1;
  const int CV = C / VEC;
  const int rows = blockDim.x / CV;
  const int cv = threadIdx.x % CV;
  const int row = threadIdx.x / CV;
  if (row >= rows) return;
  const int n = blockIdx.y;
  const long long s0 = (long long)blockIdx.x * vox_per_chunk;
  long long s1 = s0 + vox_per_chunk;
  if (s1 > spatial) s1 = spatial;
  const int c = cv * VEC;
  const h16* src;
  int pitch;
  if (c < C0) { src = x0 + (long long)n * spatial * pitch0 + c; pitch = pitch0; }
  else        { src = x1 + (long long)n * spatial * pitch1 + (c - C0); pitch = pitch1; }
  h16* dst = y + (long long)n * spatial * y_pitch + c;
  float a[VEC], b[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    a[j] = affine[((long long)n * C + c + j) * 2 + 0];
    b[j] = affine[((long long)n * C + c + j) * 2 + 1];
  }
  constexpr int U = 4;
  long long s = s0 + row;
  if constexpr (VEC == 8) {
    for (; s + (long long)(U - 1) * rows < s1; s += (long long)U * rows) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(src + (s + (long long)u * rows) * pitch));
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float f[8];
        unpack8(v[u], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float t = fmaf(f[j], a[j], b[j]);
          f[j] = gn_act(t, act);
        }
        *reinterpret_cast<uint4*>(dst + (s + (long long)u * rows) * y_pitch) = pack8(f);
      }
    }
  }
  for (; s < s1; s += rows) {
    float f[VEC];
    if constexpr (VEC == 8) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(src + s * pitch)), f);
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) f[j] = h2f(src[s * pitch + j]);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float t = fmaf(f[j], a[j], b[j]);
      f[j] = gn_act(t, act);
    }
    if constexpr (VEC == 8) {
      *reinterpret_cast<uint4*>(dst + s * y_pitch) = pack8(f);
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) dst[s * y_pitch + j] = f2h(f[j]);
    }
  }
}

// ---- single-launch GroupNorm for small tensors ---------------------------------------------------------
// The deep levels of a latent UNet normalise tensors of 10^4..10^6 elements ~50 times per step; the three-kernel form
// above (partials, finalize, apply) then costs three launch latencies for microseconds of work.  Here one CTA per
// (sample, group) owns the group's slab [spatial][cpg]: pass 1 sums it, a block reduction in fp64 gives mean / rstd,
// pass 2 re-reads it (L1 / L2 hits), normalises, applies the activation and stores.  Thread t keeps one channel
// vector (VEC channels, fixed) and strides over rows, so its affine pairs live in registers.
template <int VEC>
__device__ __forceinline__ void gn_load_vec(const h16* p, float* f) {
  if constexpr (VEC == 8) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(p)), f);
  } else if constexpr (VEC == 4) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
    const h162 lo = *reinterpret_cast<const h162*>(&v.x);
    const h162 hi = *reinterpret_cast<const h162*>(&v.y);
    f[0] = __low2float(lo); f[1] = __high2float(lo); f[2] = __low2float(hi); f[3] = __high2float(hi);
  } else if constexpr (VEC == 2) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(p));
    const h162 h = *reinterpret_cast<const h162*>(&v);
    f[0] = __low2float(h); f[1] = __high2float(h);
  } else {
    f[0] = h2f(p[0]);
  }
}
template <int VEC>
__device__ __forceinline__ void gn_store_vec(h16* p, const float* f) {
  if constexpr (VEC == 8) {
    *reinterpret_cast<uint4*>(p) = pack8(f);
  } else if constexpr (VEC == 4) {
    const h162 lo = f2h2(f[0], f[1]), hi = f2h2(f[2], f[3]);
    uint2 v;
    v.x = *reinterpret_cast<const uint32_t*>(&lo);
    v.y = *reinterpret_cast<const uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = v;
  } else if constexpr (VEC == 2) {
    const h162 h = f2h2(f[0], f[1]);
    *reinterpret_cast<uint32_t*>(p) = *reinterpret_cast<const uint32_t*>(&h);
  } else {
    p[0] = f2h(f[0]);
  }
}

// KREG > 0 (VEC == 8 only): every thread keeps its (at most KREG) row vectors in registers between the statistics and
// the normalisation, so the tensor is read once (the second pass of the KREG = 0 form re-reads it from L1 / L2 behind
// one more dependent-latency chain).
template <int VEC, int KREG = 0>
__global__ void __launch_bounds__(512) gn_fused_small_kernel(const h16* __restrict__ x0,
                                                             const h16* __restrict__ x1, int C0, int C1,
                                                             int pitch0, int pitch1, int spatial, int groups, float eps,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, int act,
                                                             h16* __restrict__ y, int y_pitch) {
  const int g = blockIdx.x, n = blockIdx.y;
  const int C = C0 + C1, cpg = C / groups;
  const int c_first = g * cpg;                       // the host guarantees a group never straddles the two sources
  const h16* src;
  int pitch;
  if (c_first < C0) { src = x0 + (long long)n * spatial * pitch0 + c_first; pitch = pitch0; }
  else              { src = x1 + (long long)n * spatial * pitch1 + (c_first - C0); pitch = pitch1; }
  h16* dst = y + (long long)n * spatial * y_pitch + c_first;
  const int vpr = cpg / VEC;                         // channel vectors per row (<= blockDim.x)
  const int rows_per_iter = blockDim.x / vpr;
  const int v = threadIdx.x % vpr, row0 = threadIdx.x / vpr;
  const bool active = row0 < rows_per_iter;
  const int c_off = v * VEC;
  const float piv = h2f(src[0]);                     // statistics pivot: the group's first element (see stats)

  float s = 0.f, q = 0.f;
  uint4 keep[KREG > 0 ? KREG : 1];
  if (active) {
    if constexpr (KREG > 0 && VEC == 8) {
#pragma unroll
      for (int k = 0; k < KREG; ++k) {
        const int r = row0 + k * rows_per_iter;
        keep[k] = r < spatial ? __ldg(reinterpret_cast<const uint4*>(src + (long long)r * pitch + c_off))
                              : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int k = 0; k < KREG; ++k) {          // same row order as the loop form: identical sums
        if (row0 + k * rows_per_iter >= spatial) continue;   // a row past the slab adds nothing (not d = -piv)
        float f[8];
        unpack8(keep[k], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = f[j] - piv;
          s += d;
          q = fmaf(d, d, q);
        }
      }
    } else {
#pragma unroll 4
      for (int r = row0; r < spatial; r += rows_per_iter) {
        float f[VEC];
        gn_load_vec<VEC>(src + (long long)r * pitch + c_off, f);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float d = f[j] - piv;
          s += d;
          q = fmaf(d, d, q);
        }
      }
    }
  }
  double ds = (double)s, dq = (double)q;
  for (int o = 16; o > 0; o >>= 1) {
    ds += __shfl_xor_sync(0xffffffffu, ds, o);
    dq += __shfl_xor_sync(0xffffffffu, dq, o);
  }
  __shared__ double red_s[16], red_q[16];
  __shared__ float stat[2];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red_s[w] = ds; red_q[w] = dq; }
  __syncthreads();
  if (w == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    ds = l < nw ? red_s[l] : 0.0;
    dq = l < nw ? red_q[l] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      ds += __shfl_xor_sync(0xffffffffu, ds, o);
      dq += __shfl_xor_sync(0xffffffffu, dq, o);
    }
    if (l == 0) {
      const double cnt = (double)spatial * cpg;
      const double dm = ds / cnt;
      double var = dq / cnt - dm * dm;
      if (var < 0.0) var = 0.0;
      stat[0] = (float)((double)piv + dm);
      stat[1] = (float)(1.0 / sqrt(var + (double)eps));
    }
  }
  __syncthreads();
  if (active) {
    const float mean = stat[0], rstd = stat[1];
    float a[VEC], b[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      a[j] = rstd * gamma[c_first + c_off + j];
      b[j] = beta[c_first + c_off + j] - mean * a[j];
    }
    if constexpr (KREG > 0 && VEC == 8) {
#pragma unroll
      for (int k = 0; k < KREG; ++k) {
        const int r = row0 + k * rows_per_iter;
        if (r < spatial) {
          float f[8];
          unpack8(keep[k], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float t = fmaf(f[j], a[j], b[j]);
            f[j] = gn_act(t, act);
          }
          gn_store_vec<8>(dst + (long long)r * y_pitch + c_off, f);
        }
      }
    } else {
#pragma unroll 4
      for (int r = row0; r < spatial; r += rows_per_iter) {
        float f[VEC];
        gn_load_vec<VEC>(src + (long long)r * pitch + c_off, f);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float t = fmaf(f[j], a[j], b[j]);
          f[j] = gn_act(t, act);
        }
        gn_store_vec<VEC>(dst + (long long)r * y_pitch + c_off, f);
      }
    }
  }
  // pad channels [C, y_pitch) stay exact zeros for the consumers' vector loads: the last group's CTA writes them
  if (y_pitch > C && g == groups - 1) {
    const int padw = y_pitch - C;
    h16* pad = y + (long long)n * spatial * y_pitch + C;
    for (int i = threadIdx.x; i < spatial * padw; i += blockDim.x)
      pad[(long long)(i / padw) * y_pitch + (i % padw)] = f2h(0.f);
  }
}

// zero the pad channels [C, pitch) of a channels-last tensor (only when pitch > C)
__global__ void zero_pad_channels_kernel(h16* y, long long rows, int C, int pitch) {
  const int padw = pitch - C;
  const long long total = rows * padw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    y[(idx / padw) * pitch + C + idx % padw] = f2h(0.f);
  }
}


// ---- SPADE modulation -----------------------------------------------------------------------------
// one thread per (voxel, 8-channel vector) when everything is 16-byte aligned, else per (voxel, channel)
template <int VEC>
__global__ void spade_apply_kernel(const h16* __restrict__ x0, const h16* __restrict__ x1, int C0,
                                   int C1, int pitch0, int pitch1, long long spatial, int N,
                                   const float* __restrict__ affine, const h16* __restrict__ gb, int gb_pitch,
                                   const float* __restrict__ gb_affine, int act, h16* __restrict__ y,
                                   int y_pitch) {
  const int C = C0 + C1;
  const int CV = C / VEC;
  const long long total = (long long)N * spatial * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % CV) * VEC;
    const long long row = i / CV;
    const int n = (int)(row / spatial);
    const h16* src = c < C0 ? x0 + row * pitch0 + c : x1 + row * pitch1 + (c - C0);
    const h16* g = gb + row * gb_pitch + c;
    float xv[VEC], gv[VEC], tv[VEC];
    if constexpr (VEC == 8) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(src)), xv);
      unpack8(__ldg(reinterpret_cast<const uint4*>(g)), gv);
      unpack8(__ldg(reinterpret_cast<const uint4*>(g + C)), tv);
    } else {
      xv[0] = h2f(src[0]); gv[0] = h2f(g[0]); tv[0] = h2f(g[C]);
    }
    const float* ax = affine + ((long long)n * C + c) * 2;
    const float* ag = gb_affine + ((long long)n * 2 * C + c) * 2;
    const float* at = gb_affine + ((long long)n * 2 * C + C + c) * 2;
    float out[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float nx = fmaf(xv[j], ax[2 * j], ax[2 * j + 1]);
      const float gg = fmaf(gv[j], ag[2 * j], ag[2 * j + 1]);
      const float tt = fmaf(tv[j], at[2 * j], at[2 * j + 1]);
      out[j] = apply_act(fmaf(nx, 1.0f + gg, tt), act);
    }
    h16* dst = y + row * y_pitch + c;
    if constexpr (VEC == 8) *reinterpret_cast<uint4*>(dst) = pack8(out);
    else dst[0] = f2h(out[0]);
  }
}

// ---- LayerNorm: one warp per row ----------------------------------------------------------------
__global__ void layernorm_kernel(const h16* __restrict__ x, long long M, int C, int x_pitch,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 h16* __restrict__ y, int y_pitch) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const h16* xr = x + row * x_pitch;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += h2f(xr[c]);
  const float mean = warp_sum(s) / C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = h2f(xr[c]) - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  h16* yr = y + row * y_pitch;
  for (int c = lane; c < C; c += 32) {
    const float v = (h2f(xr[c]) - mean) * rstd * gamma[c] + beta[c];
    yr[c] = f2h(v);
  }
  for (int c = C + lane; c < y_pitch; c += 32) yr[c] = f2h(0.f);
}

// 128-bit variant (C % 8 == 0, 16-byte-aligned rows): the row lives in registers (VPL vectors of 8 channels per lane),
// one global read and one write per element instead of three scalar reads; mean and variance as in the scalar kernel
// (two passes, fp32), the per-lane summation order differs.
template <int VPL>
__global__ void layernorm_vec_kernel(const h16* __restrict__ x, long long M, int C, int x_pitch,
                                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                     h16* __restrict__ y, int y_pitch) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * x_pitch);
  float f[VPL][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + 32 * i;
    if (vi < nv) {
      const uint4 t = __ldg(xr + vi);
      unpack8(t, f[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[i][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[i][j] = 0.f;
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    if (lane + 32 * i < nv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[i][j] - mean;
        q = fmaf(d, d, q);
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  h16* yr = y + row * y_pitch;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + 32 * i;
    if (vi < nv) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * vi);
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * vi + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * vi);
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * vi + 1);
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (f[i][j] - mean) * rstd * g[j] + b[j];
      *reinterpret_cast<uint4*>(yr + vi * 8) = pack8(v);
    }
  }
  for (int c = C + lane; c < y_pitch; c += 32) yr[c] = f2h(0.f);
}

static int gn_chunks(int N, long long spatial, int rows) {
  long long want = (4ll * sm_count() + N - 1) / N;
  long long maxc = (spatial + rows * 8 - 1) / (rows * 8);   // at least 8 iterations per thread
  if (maxc < 1) maxc = 1;
  long long c = want < maxc ? want : maxc;
  if (c > kGnMaxChunks) c = kGnMaxChunks;
  if (c < 1) c = 1;
  return (int)c;
}

static void gn_block_shape(int C, bool vec_ok, int& vec, int& cv, int& rows) {
  vec = vec_ok ? 8 : 1;
  cv = C / vec;
  rows = 256 / cv;
  if (rows < 1) rows = 1;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_groupnorm_workspace_bytes(int32_t N, int64_t spatial, int32_t C_total) {
  (void)spatial;
  return (int64_t)N * kGnMaxChunks * C_total * 2 * sizeof(float);
}

extern "C" int b200_groupnorm_stats(const b200_gn_stats_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->x_ptr[0] && p->gamma && p->beta && p->partial && p->affine, "gn_stats: null pointer");
  const int C0 = p->x_C[0], C1 = p->x_ptr[1] ? p->x_C[1] : 0;
  const int C = C0 + C1;
  B200_CHECK_ARG(p->groups >= 1 && C % p->groups == 0, "gn_stats: %d channels not divisible by %d groups", C, p->groups);
  B200_CHECK_ARG(p->N >= 1 && p->spatial >= 1, "gn_stats: empty input");
  int vec, cv, rows;
  const bool vec_ok = C0 % 8 == 0 && C1 % 8 == 0 && p->x_pitch[0] % 8 == 0 && (C1 == 0 || p->x_pitch[1] % 8 == 0) &&
                      ((uintptr_t)p->x_ptr[0] % 16 == 0) && (C1 == 0 || (uintptr_t)p->x_ptr[1] % 16 == 0);
  gn_block_shape(C, vec_ok, vec, cv, rows);
  B200_CHECK_ARG(cv <= 1024, "gn_stats: too many channels (%d)", C);
  const size_t smem = (size_t)rows * C * 2 * sizeof(float);
  B200_CHECK_ARG(smem <= 48 * 1024, "gn_stats: %d channels need %zu bytes of shared memory (at most 6144 channels)", C,
                 smem);
  const int chunks = gn_chunks(p->N, p->spatial, rows);
  const long long vpc = (p->spatial + chunks - 1) / chunks;
  const int threads = cv * rows;
  const int cpg = C / p->groups;
  dim3 grid(chunks, p->N);
  const h16* x0 = reinterpret_cast<const h16*>(p->x_ptr[0]);
  const h16* x1 = reinterpret_cast<const h16*>(p->x_ptr[1]);
  if (vec == 8)
    B200_CUDA(b200::launch_kernel(gn_partial_kernel<8>, grid, threads, smem, stream, x0, x1, C0, C1, p->x_pitch[0], p->x_pitch[1], p->spatial, cpg, vpc, p->partial));
  else
    B200_CUDA(b200::launch_kernel(gn_partial_kernel<1>, grid, threads, smem, stream, x0, x1, C0, C1, p->x_pitch[0], p->x_pitch[1], p->spatial, cpg, vpc, p->partial));
  B200_LAUNCH_CHECK("gn_partial_kernel");
  B200_CUDA(b200::launch_kernel(gn_finalize_kernel, dim3(p->groups, p->N), 128, 0, stream, p->partial, x0, x1, C0, p->x_pitch[0], p->x_pitch[1], chunks, C, p->groups, p->spatial, p->eps,
                                                                p->gamma, p->beta, p->affine));
  B200_LAUNCH_CHECK("gn_finalize_kernel");
  return B200_OK;
}

extern "C" int b200_groupnorm_from_partials_ex(const b200_gn_stats_params* p, const float* const partial[2],
                                               const int32_t slots[2], const int32_t group[2], void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && partial && slots && partial[0] && p->gamma && p->beta && p->affine, "groupnorm_from_partials: null pointer");
  const int C0 = p->x_C[0], C1 = partial[1] ? p->x_C[1] : 0;
  const int C = C0 + C1;
  B200_CHECK_ARG(p->N >= 1 && p->spatial >= 1 && p->groups >= 1 && C % p->groups == 0, "groupnorm_from_partials: bad shape");
  const int cpg = C / p->groups;
  const int g0 = (group && group[0]) ? group[0] : 8, g1 = (group && C1 && group[1]) ? group[1] : 8;
  B200_CHECK_ARG((g0 == 8 || g0 == 4) && (g1 == 8 || g1 == 4), "groupnorm_from_partials: producer groups are 8 or 4 channels wide");
  B200_CHECK_ARG(cpg % g0 == 0 && (!C1 || cpg % g1 == 0) && C0 % cpg == 0 && C0 % g0 == 0 && C1 % g1 == 0 && slots[0] >= 1 &&
                     (!C1 || slots[1] >= 1),
                 "groupnorm_from_partials: groups of %d channels do not tile the %d / %d-channel partials", cpg, g0, g1);
  dim3 grid(p->groups, p->N);
  B200_CUDA(b200::launch_kernel(gn_finalize_partials_kernel, grid, 256, 0, stream, partial[0], partial[1], slots[0], C1 ? slots[1] : 0, C0, C1,
                                                        g0 == 4 ? 2 : 3, g1 == 4 ? 2 : 3, p->groups, p->spatial, p->eps, p->gamma, p->beta,
                                                        p->affine));
  B200_LAUNCH_CHECK("gn_finalize_partials_kernel");
  return B200_OK;
}

extern "C" int b200_groupnorm_apply(const b200_gn_apply_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->x_ptr[0] && p->affine && p->y_ptr, "gn_apply: null pointer");
  const int C0 = p->x_C[0], C1 = p->x_ptr[1] ? p->x_C[1] : 0;
  const int C = C0 + C1;
  B200_CHECK_ARG(p->y_pitch >= C, "gn_apply: y_pitch %d < C %d", p->y_pitch, C);
  B200_CHECK_ARG(gn_act_ok(p->act), "gn_apply: unsupported activation %d", p->act);
  const int vec = (C0 % 8 == 0 && C1 % 8 == 0 && p->x_pitch[0] % 8 == 0 && (C1 == 0 || p->x_pitch[1] % 8 == 0) &&
                   p->y_pitch % 8 == 0 && ((uintptr_t)p->x_ptr[0] % 16 == 0) &&
                   (C1 == 0 || (uintptr_t)p->x_ptr[1] % 16 == 0) && ((uintptr_t)p->y_ptr % 16 == 0)) ? 8 : 1;
  int cv = C / vec;
  B200_CHECK_ARG(cv <= 1024, "gn_apply: too many channels (%d)", C);
  int rows = 256 / cv;
  if (rows < 1) rows = 1;
  // enough slabs to fill the machine a few times over, but at least ~16 voxels per thread
  long long chunks = (8ll * sm_count() + p->N - 1) / p->N;
  const long long maxc = (p->spatial + (long long)rows * 16 - 1) / ((long long)rows * 16);
  if (chunks > maxc) chunks = maxc;
  if (chunks < 1) chunks = 1;
  const long long vpc = (p->spatial + chunks - 1) / chunks;
  dim3 grid((unsigned)chunks, p->N);
  const int threads = cv * rows;
  const h16* x0 = reinterpret_cast<const h16*>(p->x_ptr[0]);
  const h16* x1 = reinterpret_cast<const h16*>(p->x_ptr[1]);
  h16* y = reinterpret_cast<h16*>(p->y_ptr);
  if (vec == 8)
    B200_CUDA(b200::launch_kernel(gn_apply_kernel<8>, grid, threads, 0, stream, x0, x1, C0, C1, p->x_pitch[0], p->x_pitch[1], p->spatial, vpc, p->affine, p->act, y, p->y_pitch));
  else
    B200_CUDA(b200::launch_kernel(gn_apply_kernel<1>, grid, threads, 0, stream, x0, x1, C0, C1, p->x_pitch[0], p->x_pitch[1], p->spatial, vpc, p->affine, p->act, y, p->y_pitch));
  B200_LAUNCH_CHECK("gn_apply_kernel");
  if (p->y_pitch > C) {
    const long long rows = (long long)p->N * p->spatial;
    long long zb = (rows * (p->y_pitch - C) + 255) / 256;
    if (zb > 4ll * sm_count()) zb = 4ll * sm_count();
    B200_CUDA(b200::launch_kernel(zero_pad_channels_kernel, (unsigned)zb, 256, 0, stream, y, rows, C, p->y_pitch));
    B200_LAUNCH_CHECK("zero_pad_channels_kernel");
  }
  return B200_OK;
}

extern "C" int b200_groupnorm_fused(const b200_gn_stats_params* sp, const b200_gn_apply_params* ap, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(sp && ap && sp->x_ptr[0] && sp->gamma && sp->beta && ap->y_ptr, "groupnorm_fused: null pointer");
  const int C0 = sp->x_C[0], C1 = sp->x_ptr[1] ? sp->x_C[1] : 0;
  const int C = C0 + C1;
  B200_CHECK_ARG(sp->groups >= 1 && C % sp->groups == 0, "groupnorm_fused: %d channels not divisible by %d groups", C,
                 sp->groups);
  B200_CHECK_ARG(sp->N >= 1 && sp->N <= 65535 && sp->spatial >= 1 && sp->spatial < (1ll << 24),
                 "groupnorm_fused: batch / spatial extent out of range");
  B200_CHECK_ARG(ap->y_pitch >= C, "groupnorm_fused: y_pitch %d < C %d", ap->y_pitch, C);
  B200_CHECK_ARG(gn_act_ok(ap->act), "groupnorm_fused: unsupported activation %d", ap->act);
  const int cpg = C / sp->groups;
  B200_CHECK_ARG(C1 == 0 || C0 % cpg == 0, "groupnorm_fused: a group of %d channels straddles the two sources", cpg);
  // widest vector every access of every group can use: channel offsets, row pitches and base addresses
  auto ok = [&](int vec) {
    if (cpg % vec) return false;
    const uintptr_t bytes = (uintptr_t)vec * 2;
    if (sp->x_pitch[0] % vec || ap->y_pitch % vec || (C1 && sp->x_pitch[1] % vec)) return false;
    if ((uintptr_t)sp->x_ptr[0] % bytes || (uintptr_t)ap->y_ptr % bytes) return false;
    if (C1 && (uintptr_t)sp->x_ptr[1] % bytes) return false;
    return true;
  };
  const int vec = ok(8) ? 8 : ok(4) ? 4 : ok(2) ? 2 : 1;
  B200_CHECK_ARG(cpg / vec <= 512, "groupnorm_fused: %d channels per group is too many for one CTA", cpg);
  const h16* x0 = reinterpret_cast<const h16*>(sp->x_ptr[0]);
  const h16* x1 = reinterpret_cast<const h16*>(sp->x_ptr[1]);
  h16* y = reinterpret_cast<h16*>(ap->y_ptr);
  dim3 grid(sp->groups, sp->N);
#define B200_GN_FUSED(V)                                                                                           \
  B200_CUDA(b200::launch_kernel(gn_fused_small_kernel<V>, grid, 512, 0, stream, x0, x1, C0, C1, sp->x_pitch[0], sp->x_pitch[1], (int)sp->spatial, \
                                                     sp->groups, sp->eps, sp->gamma, sp->beta, ap->act, y, ap->y_pitch))
  if (vec == 8) {
    // rows each thread visits: 512 threads / (cpg / 8) vectors per row
    const int rows_per_iter = 512 / (cpg / 8);
    const long long iters = (sp->spatial + rows_per_iter - 1) / rows_per_iter;
#define B200_GN_FUSED_K(K)                                                                                          \
  B200_CUDA(b200::launch_kernel(gn_fused_small_kernel<8, K>, grid, 512, 0, stream, x0, x1, C0, C1, sp->x_pitch[0], sp->x_pitch[1], (int)sp->spatial, \
                                                     sp->groups, sp->eps, sp->gamma, sp->beta, ap->act, y, ap->y_pitch))
    if (iters <= 2) B200_GN_FUSED_K(2);
    else if (iters <= 4) B200_GN_FUSED_K(4);
    else if (iters <= 8) B200_GN_FUSED_K(8);
    else B200_GN_FUSED(8);
#undef B200_GN_FUSED_K
  }
  else if (vec == 4) B200_GN_FUSED(4);
  else if (vec == 2) B200_GN_FUSED(2);
  else B200_GN_FUSED(1);
#undef B200_GN_FUSED
  B200_LAUNCH_CHECK("gn_fused_small_kernel");
  return B200_OK;
}

extern "C" int b200_spade_apply(const b200_gn_apply_params* p, const void* gb, int32_t gb_pitch, const float* gb_affine,
                                void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->x_ptr[0] && p->affine && p->y_ptr && gb && gb_affine, "spade_apply: null pointer");
  const int C0 = p->x_C[0], C1 = p->x_ptr[1] ? p->x_C[1] : 0;
  const int C = C0 + C1;
  B200_CHECK_ARG(p->y_pitch >= C && gb_pitch >= 2 * C && p->N >= 1 && p->spatial >= 1, "spade_apply: bad shape");
  const bool vec = C0 % 8 == 0 && C1 % 8 == 0 && p->x_pitch[0] % 8 == 0 && (C1 == 0 || p->x_pitch[1] % 8 == 0) &&
                   p->y_pitch % 8 == 0 && gb_pitch % 8 == 0 && ((uintptr_t)p->x_ptr[0] % 16 == 0) &&
                   (C1 == 0 || (uintptr_t)p->x_ptr[1] % 16 == 0) && ((uintptr_t)p->y_ptr % 16 == 0) &&
                   ((uintptr_t)gb % 16 == 0);
  const long long total = (long long)p->N * p->spatial * (C / (vec ? 8 : 1));
  long long blocks = (total + 255) / 256;
  if (blocks > 16ll * sm_count()) blocks = 16ll * sm_count();
  const h16* x0 = reinterpret_cast<const h16*>(p->x_ptr[0]);
  const h16* x1 = reinterpret_cast<const h16*>(p->x_ptr[1]);
  const h16* g = reinterpret_cast<const h16*>(gb);
  h16* y = reinterpret_cast<h16*>(p->y_ptr);
  if (vec)
    B200_CUDA(b200::launch_kernel(spade_apply_kernel<8>, (unsigned)blocks, 256, 0, stream, x0, x1, C0, C1, p->x_pitch[0], p->x_pitch[1], p->spatial,
                                                                p->N, p->affine, g, gb_pitch, gb_affine, p->act, y, p->y_pitch));
  else
    B200_CUDA(b200::launch_kernel(spade_apply_kernel<1>, (unsigned)blocks, 256, 0, stream, x0, x1, C0, C1, p->x_pitch[0], p->x_pitch[1], p->spatial,
                                                                p->N, p->affine, g, gb_pitch, gb_affine, p->act, y, p->y_pitch));
  B200_LAUNCH_CHECK("spade_apply_kernel");
  if (p->y_pitch > C) {
    const long long rows = (long long)p->N * p->spatial;
    long long zb = (rows * (p->y_pitch - C) + 255) / 256;
    if (zb > 4ll * sm_count()) zb = 4ll * sm_count();
    B200_CUDA(b200::launch_kernel(zero_pad_channels_kernel, (unsigned)zb, 256, 0, stream, y, rows, C, p->y_pitch));
    B200_LAUNCH_CHECK("zero_pad_channels_kernel");
  }
  return B200_OK;
}

extern "C" int b200_layernorm(const void* x, int64_t M, int32_t C, int32_t x_pitch, const float* gamma,
                              const float* beta, float eps, void* y, int32_t y_pitch, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(x && y && gamma && beta && M >= 1 && C >= 1, "layernorm: bad arguments");
  const int wpb = 8;
  const long long blocks = (M + wpb - 1) / wpb;
  B200_CHECK_ARG(blocks < (1ll << 31), "layernorm: too many rows");
  const bool vec = C % 8 == 0 && C <= 2048 && x_pitch % 8 == 0 && y_pitch % 8 == 0 && ((uintptr_t)x % 16 == 0) &&
                   ((uintptr_t)y % 16 == 0) && ((uintptr_t)gamma % 16 == 0) && ((uintptr_t)beta % 16 == 0);
#define B200_LN_LAUNCH(K)                                                                                              \
  B200_CUDA(b200::launch_kernel(K, (unsigned)blocks, wpb * 32, 0, stream, reinterpret_cast<const h16*>(x), M, C, x_pitch, \
                             gamma, beta, eps, reinterpret_cast<h16*>(y), y_pitch))
  if (!vec) B200_LN_LAUNCH(layernorm_kernel);
  else if (C <= 256) B200_LN_LAUNCH(layernorm_vec_kernel<1>);
  else if (C <= 512) B200_LN_LAUNCH(layernorm_vec_kernel<2>);
  else if (C <= 1024) B200_LN_LAUNCH(layernorm_vec_kernel<4>);
  else B200_LN_LAUNCH(layernorm_vec_kernel<8>);
#undef B200_LN_LAUNCH
  B200_LAUNCH_CHECK("layernorm_kernel");
  return B200_OK;
}
