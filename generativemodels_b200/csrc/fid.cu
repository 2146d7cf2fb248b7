// FIDMetric (generative/metrics/fid.py of the reference) in fp64 on the GPU: the feature moments, an fp64 tensor-core
// GEMM (DMMA, mma.m16n8k16.f64) for the Gram and the M products, pivoted Cholesky, Householder tridiagonalisation,
// Sturm bisection and the finish.  Contracts: include/b200gen_fid.h.
#include <math_constants.h>

#include <algorithm>
#include <cfloat>
#include <climits>

#include "common.cuh"
#include "../../include/b200gen_fid.h"

namespace b200 {
namespace {

constexpr double kEps = 2.220446049250313e-16;  // 2^-52
constexpr int kRed = 1024;                      // threads of the one-CTA kernels

// ---------------------------------------------------------------------------------------------------------------
// Fixed-order block reductions (blockDim.x == kRed): warp butterflies, then warp 0 over the 32 warp values.
// The result is valid in every thread.
__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = red[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  return red[0];
}

__device__ double block_minmax(double v, double* red, bool is_max) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmax(v, u) : fmin(v, u);
  }
  __syncthreads();
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = red[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double u = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_max ? fmax(v, u) : fmin(v, u);
    }
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  return red[0];
}

// ---------------------------------------------------------------------------------------------------------------
// Moments: column means.  A CTA of 32 x 16 threads owns 32 features; thread (f, g) sums rows g, g + 16, ... in order,
// then row 0 of the CTA adds the 16 partial sums in order.
__global__ void __launch_bounds__(512) fid_colmean_kernel(const void* x, int dt, int64_t s_row, int64_t s_col, int64_t n,
                                                          int F, double* mu) {
  __shared__ double part[16][33];
  const int f = blockIdx.x * 32 + threadIdx.x;
  double acc = 0.0;
  if (f < F)
    for (int64_t r = threadIdx.y; r < n; r += 16) acc += load_any_f64(x, dt, r * s_row + f * s_col);
  part[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && f < F) {
    double s = 0.0;
    for (int g = 0; g < 16; ++g) s += part[g][threadIdx.x];
    mu[f] = s / (double)n;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// fp64 GEMM on the tensor cores: C[m][n] = alpha * sum_k opA[m][k] * opB[k][n], with opA[m][k] = A[m * s0 + k * s1]
// (minus mu[m] when mu is set) and opB[k][n] = B[k * s0 + n * s1] (minus mu[n]); out-of-range elements are zero.
// 64 x 64 CTA tile, k-step 16, 8 warps of 32 x 16 (2 x 2 m16n8k16 tiles).  sym: only tiles on or below the diagonal
// run and each value with m >= n is stored at (m, n) and (n, m), so C is symmetric to the bit.
struct Operand {
  const void* p;
  int dt;
  int fast0;           // 1: consecutive threads load consecutive indices of the first (m or k) dimension
  int64_t s0, s1;
  const double* mu;
};
struct GemmArgs {
  Operand a, b;
  int M, N;
  int64_t K;
  double alpha;
  double* c;
  int64_t ldc;
  int sym;
};

constexpr int kBM = 64, kBN = 64, kBK = 16, kPad = 4, kGemmThreads = 256;

__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// element e of a 64 (outer) x 16 (k) tile -> (outer index, k); `outer_fast` picks which of the two varies fastest
__device__ __forceinline__ void tile_coord(int e, bool outer_fast, int& o, int& k) {
  if (outer_fast) {
    o = e % 64;
    k = e / 64;
  } else {
    k = e % 16;
    o = e / 16;
  }
}

__global__ void __launch_bounds__(kGemmThreads) fid_dgemm_kernel(const GemmArgs g) {
  const int bm = blockIdx.y, bn = blockIdx.x;
  if (g.sym && bm < bn) return;
  __shared__ double As[kBK][kBM + kPad];
  __shared__ double Bs[kBK][kBN + kPad];
  const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32;
  const int wm = warp / 4, wn = warp % 4, grp = lane / 4, tig = lane % 4;
  const int m0 = bm * kBM, n0 = bn * kBN;
  double acc[2][2][4] = {};
  for (int64_t k0 = 0; k0 < g.K; k0 += kBK) {
#pragma unroll
    for (int r = 0; r < (kBM * kBK) / kGemmThreads; ++r) {
      const int e = tid + r * kGemmThreads;
      int o, k;
      tile_coord(e, g.a.fast0 != 0, o, k);  // A's first index is m: fast0 means m fastest
      const int m = m0 + o;
      const int64_t kk = k0 + k;
      double v = 0.0;
      if (m < g.M && kk < g.K) {
        v = load_any_f64(g.a.p, g.a.dt, (int64_t)m * g.a.s0 + kk * g.a.s1);
        if (g.a.mu) v -= g.a.mu[m];
      }
      As[k][o] = v;
      tile_coord(e, g.b.fast0 == 0, o, k);  // B's first index is k: fast0 means k fastest
      const int n = n0 + o;
      const int64_t kb = k0 + k;
      double w = 0.0;
      if (n < g.N && kb < g.K) {
        w = load_any_f64(g.b.p, g.b.dt, kb * g.b.s0 + (int64_t)n * g.b.s1);
        if (g.b.mu) w -= g.b.mu[n];
      }
      Bs[k][o] = w;
    }
    __syncthreads();
    double af[2][8], bf[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 8; ++i) af[mt][i] = As[tig + 4 * (i >> 1)][wm * 32 + mt * 16 + grp + 8 * (i & 1)];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) bf[nt][i] = Bs[tig + 4 * i][wn * 16 + nt * 8 + grp];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) dmma16816(acc[mt][nt], af[mt], bf[nt]);
    __syncthreads();
  }
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = m0 + wm * 32 + mt * 16 + grp + 8 * (i >> 1);
        const int n = n0 + wn * 16 + nt * 8 + 2 * tig + (i & 1);
        if (m >= g.M || n >= g.N) continue;
        const double v = g.alpha * acc[mt][nt][i];
        if (!g.sym) {
          g.c[(int64_t)m * g.ldc + n] = v;
        } else if (m >= n) {
          g.c[(int64_t)m * g.ldc + n] = v;
          g.c[(int64_t)n * g.ldc + m] = v;
        }
      }
}

cudaError_t dgemm(const GemmArgs& g, cudaStream_t stream) {
  const dim3 grid((g.N + kBN - 1) / kBN, (g.M + kBM - 1) / kBM);
  return launch_kernel(fid_dgemm_kernel, grid, dim3(kGemmThreads), 0, stream, g);
}

// ---------------------------------------------------------------------------------------------------------------
// Frechet distance.  Workspace (doubles): W [F][F] (the factor's working copy of sigma_y, then T = sigma_x G),
// G [F][F], M [F][F], d, e, v, pw, eig [F] each, State, chosen [F] int32.
struct State {
  double tol, piv_sqrt, tau, glo, ghi, pivmin;
  int32_t piv, stop, rank, nonfinite;
};

struct Ws {
  double *W, *G, *M, *d, *e, *v, *pw, *eig;
  State* st;
  int32_t* chosen;
};

Ws carve(double* base, int F, double* eig_out) {
  const size_t F2 = (size_t)F * F;
  Ws w;
  w.W = base;
  w.G = w.W + F2;
  w.M = w.G + F2;
  w.d = w.M + F2;
  w.e = w.d + F;
  w.v = w.e + F;
  w.pw = w.v + F;
  w.eig = w.pw + F;
  w.st = reinterpret_cast<State*>(w.eig + F);
  w.chosen = reinterpret_cast<int32_t*>(w.st + 1);
  if (eig_out) w.eig = eig_out;
  return w;
}

int64_t ws_bytes(int F) {
  return (int64_t)(3 * (int64_t)F * F + 5 * (int64_t)F) * 8 + (int64_t)sizeof(State) + 4 * (int64_t)F;
}

// W = sigma_y, G = 0 (elementwise over F * F)
__global__ void __launch_bounds__(256) fid_chol_fill_kernel(const double* sy, double* W, double* G, int64_t F2) {
  for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < F2; i += (int64_t)gridDim.x * 256) {
    W[i] = sy[i];
    G[i] = 0.0;
  }
}

// tol = F eps max(diag sigma_y) (not-a-number entries ignored), nothing chosen, rank 0
__global__ void __launch_bounds__(kRed) fid_chol_init_kernel(const double* sy, int F, State* st, int32_t* chosen) {
  __shared__ double red[32];
  double mx = 0.0;
  for (int i = threadIdx.x; i < F; i += kRed) {
    chosen[i] = 0;
    const double v = sy[(int64_t)i * F + i];
    if (v > mx) mx = v;
  }
  mx = block_minmax(mx, red, true);
  if (threadIdx.x == 0) {
    st->tol = (double)F * kEps * mx;
    st->stop = 0;
    st->rank = 0;
    st->piv = 0;
    st->piv_sqrt = 1.0;
  }
}

// step j: the largest remaining diagonal entry among features not chosen (lowest index on a tie); stop when it is
// <= tol or not a number
__global__ void __launch_bounds__(kRed) fid_chol_pivot_kernel(const double* W, int F, int j, State* st,
                                                              int32_t* chosen) {
  __shared__ double sv[32];
  __shared__ int si[32];
  if (st->stop) return;
  double best = -DBL_MAX;
  int bi = INT_MAX;
  for (int i = threadIdx.x; i < F; i += kRed) {
    if (chosen[i]) continue;
    const double v = W[(int64_t)i * F + i];
    if (v > best || (v == best && i < bi)) {
      best = v;
      bi = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double v = __shfl_xor_sync(0xffffffffu, best, o);
    const int i = __shfl_xor_sync(0xffffffffu, bi, o);
    if (v > best || (v == best && i < bi)) {
      best = v;
      bi = i;
    }
  }
  if (threadIdx.x % 32 == 0) {
    sv[threadIdx.x / 32] = best;
    si[threadIdx.x / 32] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kRed / 32; ++w)
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) {
        best = sv[w];
        bi = si[w];
      }
    if (!(best > st->tol) || bi == INT_MAX) {
      st->stop = 1;
    } else {
      st->piv = bi;
      st->piv_sqrt = sqrt(best);
      st->rank = j + 1;
      chosen[bi] = 1;
    }
  }
}

// step j: column j of G and the rank-1 update of the features not chosen, W[i][k] -= g_i g_k with g = W[p][.] / d;
// a CTA owns 256 columns of 8 rows.  Row p is not written in this step.
__global__ void __launch_bounds__(256) fid_chol_update_kernel(double* W, double* G, int F, int j, const State* st,
                                                              const int32_t* chosen) {
  if (st->stop) return;
  const int p = st->piv;
  const double d = st->piv_sqrt;
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k >= F) return;
  const double* wp = W + (int64_t)p * F;
  const bool kc = chosen[k];
  const double gk = wp[k] / d;
  for (int r = 0; r < 8; ++r) {
    const int i = blockIdx.y * 8 + r;
    if (i >= F) break;
    if (k == 0) G[(int64_t)i * F + j] = i == p ? d : (chosen[i] ? 0.0 : wp[i] / d);
    if (kc || chosen[i]) continue;
    W[(int64_t)i * F + k] -= (wp[i] / d) * gk;
  }
}

// Tridiagonalisation, step k: the reflector H = I - tau v v^T (v[k+1] = 1) that zeroes M[k+2..F-1][k]
// (dlarfg without its rescaling), d[k] = M[k][k], e[k] = beta.
__global__ void __launch_bounds__(kRed) fid_house_kernel(const double* M, int F, int k, double* d, double* e, double* v,
                                                         State* st) {
  __shared__ double red[32];
  const double* col = M + (int64_t)k * F;  // row k == column k (M is symmetric)
  double s = 0.0;
  for (int i = k + 2 + threadIdx.x; i < F; i += kRed) s += col[i] * col[i];
  const double xnorm2 = block_sum(s, red);
  const double alpha = col[k + 1];
  double beta = alpha, tau = 0.0, scale = 0.0;
  if (xnorm2 != 0.0) {
    beta = -copysign(sqrt(alpha * alpha + xnorm2), alpha);
    tau = (beta - alpha) / beta;
    scale = 1.0 / (alpha - beta);
  }
  for (int i = k + 2 + threadIdx.x; i < F; i += kRed) v[i] = col[i] * scale;
  if (threadIdx.x == 0) {
    v[k + 1] = 1.0;
    d[k] = M[(int64_t)k * F + k];
    e[k] = beta;
    st->tau = tau;
  }
}

// p[i] = tau * sum_j M[i][j] v[j] over the trailing block, one warp per row
__global__ void __launch_bounds__(256) fid_symv_kernel(const double* M, int F, int k, const double* v, double* pw,
                                                       const State* st) {
  const int i = k + 1 + blockIdx.x * 8 + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (i >= F) return;
  const double* row = M + (int64_t)i * F;
  double s = 0.0;
  for (int j = k + 1 + lane; j < F; j += 32) s += row[j] * v[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) pw[i] = st->tau * s;
}

// w = p - (tau / 2) (p^T v) v, in place of p
__global__ void __launch_bounds__(kRed) fid_house_w_kernel(int F, int k, const double* v, double* pw,
                                                           const State* st) {
  __shared__ double red[32];
  double s = 0.0;
  for (int i = k + 1 + threadIdx.x; i < F; i += kRed) s += pw[i] * v[i];
  const double K = 0.5 * st->tau * block_sum(s, red);
  for (int i = k + 1 + threadIdx.x; i < F; i += kRed) pw[i] -= K * v[i];
}

// M[i][j] -= v_i w_j + w_i v_j on the trailing block; the two products are rounded separately and added, so the
// update keeps M symmetric to the bit
__global__ void __launch_bounds__(256) fid_rank2_kernel(double* M, int F, int k, const double* v, const double* w) {
  const int j = k + 1 + blockIdx.x * 256 + threadIdx.x;
  if (j >= F) return;
  const double vj = v[j], wj = w[j];
  for (int r = 0; r < 8; ++r) {
    const int i = k + 1 + blockIdx.y * 8 + r;
    if (i >= F) break;
    const double a = __dmul_rn(v[i], wj), b = __dmul_rn(w[i], vj);
    M[(int64_t)i * F + j] -= __dadd_rn(a, b);
  }
}

// the last one or two diagonal entries and the last off-diagonal one, then the Gershgorin interval, pivmin and whether
// the tridiagonal holds a non-finite value
__global__ void __launch_bounds__(kRed) fid_tri_tail_kernel(const double* M, int F, double* d, double* e, State* st) {
  __shared__ double red[32];
  if (threadIdx.x == 0) {
    if (F >= 2) {
      d[F - 2] = M[(int64_t)(F - 2) * F + F - 2];
      e[F - 2] = M[(int64_t)(F - 1) * F + F - 2];
    }
    d[F - 1] = M[(int64_t)(F - 1) * F + F - 1];
  }
  __syncthreads();
  double lo = DBL_MAX, hi = -DBL_MAX, e2 = 0.0, bad = 0.0;
  for (int i = threadIdx.x; i < F; i += kRed) {
    const double el = i > 0 ? fabs(e[i - 1]) : 0.0, er = i < F - 1 ? fabs(e[i]) : 0.0;
    if (!isfinite(d[i]) || !isfinite(el) || !isfinite(er)) bad = 1.0;
    lo = fmin(lo, d[i] - el - er);
    hi = fmax(hi, d[i] + el + er);
    e2 = fmax(e2, er * er);
  }
  lo = block_minmax(lo, red, false);
  hi = block_minmax(hi, red, true);
  e2 = block_minmax(e2, red, true);
  bad = block_minmax(bad, red, true);
  if (threadIdx.x == 0) {
    const double tnorm = fmax(fabs(lo), fabs(hi));
    const double pivmin = DBL_MIN * fmax(1.0, e2);
    const double pad = 2.0 * kEps * tnorm * F + 2.0 * pivmin;
    st->glo = lo - pad;
    st->ghi = hi + pad;
    st->pivmin = pivmin;
    st->nonfinite = bad != 0.0;
  }
}

// number of eigenvalues of the tridiagonal (d, e) below x (Sturm count, LAPACK dlaneg's guard on tiny pivots)
__device__ int sturm_count(const double* d, const double* e, int F, double x, double pivmin) {
  double q = d[0] - x;
  if (fabs(q) < pivmin) q = -pivmin;
  int c = q < 0.0;
  for (int i = 1; i < F; ++i) {
    q = d[i] - x - e[i - 1] * e[i - 1] / q;
    if (fabs(q) < pivmin) q = -pivmin;
    c += q < 0.0;
  }
  return c;
}

// eigenvalue i (ascending) by at most 128 halvings of the Gershgorin interval
__global__ void __launch_bounds__(128) fid_bisect_kernel(const double* d, const double* e, int F, const State* st,
                                                         double* eig) {
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= F) return;
  if (st->nonfinite) {
    eig[i] = CUDART_NAN;
    return;
  }
  double lo = st->glo, hi = st->ghi;
  for (int it = 0; it < 128; ++it) {
    const double mid = 0.5 * (lo + hi);
    if (mid <= lo || mid >= hi) break;
    if (sturm_count(d, e, F, mid, st->pivmin) > i)
      hi = mid;
    else
      lo = mid;
  }
  eig[i] = 0.5 * (lo + hi);
}

// |mu_x - mu_y|^2 + tr sigma_x + tr sigma_y - 2 sum sqrt(eig_i > cutoff); a not-a-number eigenvalue is never cut
__global__ void __launch_bounds__(kRed) fid_finish_kernel(const double* mux, const double* sx, const double* muy,
                                                          const double* sy, int F, const double* eig, const State* st,
                                                          double* out, int32_t* rank) {
  __shared__ double red[32];
  const double cutoff = (double)F * kEps * eig[F - 1];
  double dm = 0.0, tx = 0.0, ty = 0.0, sq = 0.0;
  for (int i = threadIdx.x; i < F; i += kRed) {
    const double df = mux[i] - muy[i];
    dm += df * df;
    tx += sx[(int64_t)i * F + i];
    ty += sy[(int64_t)i * F + i];
    if (!(eig[i] <= cutoff)) sq += sqrt(eig[i]);
  }
  dm = block_sum(dm, red);
  tx = block_sum(tx, red);
  ty = block_sum(ty, red);
  sq = block_sum(sq, red);
  if (threadIdx.x == 0) {
    *out = dm + tx + ty - 2.0 * sq;
    if (rank) *rank = st->rank;
  }
}

bool input_dtype_ok(int dt) {
  return dt == B200_DT_F32 || dt == B200_DT_F64 || dt == B200_DT_FP16 || dt == B200_DT_BF16;
}

}  // namespace
}  // namespace b200

extern "C" int b200_fid_moments(const b200_fid_moments_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->x && p->mu && p->sigma, "fid_moments: null pointer");
  B200_CHECK_ARG(b200::input_dtype_ok(p->x_dtype), "fid_moments: unknown dtype %d", p->x_dtype);
  B200_CHECK_ARG(p->n >= 2 && p->F >= 1 && p->F <= B200_FID_MAX_F, "fid_moments: bad extents %lld x %d",
                 (long long)p->n, p->F);
  B200_CHECK_ARG(p->x_strides[0] >= 0 && p->x_strides[1] >= 0, "fid_moments: negative stride");
  const int F = p->F;
  B200_CUDA(b200::launch_kernel(b200::fid_colmean_kernel, dim3((F + 31) / 32), dim3(32, 16), 0, stream, p->x,
                                (int)p->x_dtype, p->x_strides[0], p->x_strides[1], p->n, F, p->mu));
  B200_LAUNCH_CHECK("fid_colmean_kernel");
  b200::GemmArgs g = {};
  // opA[m][k] = x[k][m] - mu[m], opB[k][n] = x[k][n] - mu[n]
  g.a = {p->x, p->x_dtype, p->x_strides[1] <= p->x_strides[0], p->x_strides[1], p->x_strides[0], p->mu};
  g.b = {p->x, p->x_dtype, p->x_strides[0] < p->x_strides[1], p->x_strides[0], p->x_strides[1], p->mu};
  g.M = g.N = F;
  g.K = p->n;
  g.alpha = 1.0 / (double)(p->n - 1);
  g.c = p->sigma;
  g.ldc = F;
  g.sym = 1;
  B200_CUDA(b200::dgemm(g, stream));
  B200_LAUNCH_CHECK("fid_dgemm_kernel");
  return B200_OK;
}

extern "C" int64_t b200_frechet_workspace_bytes(int32_t F) {
  if (F < 1 || F > B200_FID_MAX_F) return -1;
  return b200::ws_bytes(F);
}

extern "C" int b200_frechet(const b200_frechet_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p && p->mu_x && p->sigma_x && p->mu_y && p->sigma_y && p->workspace && p->out,
                 "frechet: null pointer");
  B200_CHECK_ARG(p->F >= 1 && p->F <= B200_FID_MAX_F, "frechet: F = %d outside 1..%d", p->F, B200_FID_MAX_F);
  const int F = p->F;
  const b200::Ws w = b200::carve(p->workspace, F, p->eigvals);
  using namespace b200;
  const int64_t F2 = (int64_t)F * F;
  const int fill_blocks = (int)std::min<int64_t>((F2 + 255) / 256, 4096);

  // 1. pivoted Cholesky of sigma_y: G = P L
  B200_CUDA(launch_kernel(fid_chol_fill_kernel, dim3(fill_blocks), dim3(256), 0, stream, p->sigma_y, w.W, w.G, F2));
  B200_LAUNCH_CHECK("fid_chol_fill_kernel");
  B200_CUDA(launch_kernel(fid_chol_init_kernel, dim3(1), dim3(kRed), 0, stream, p->sigma_y, F, w.st, w.chosen));
  B200_LAUNCH_CHECK("fid_chol_init_kernel");
  const dim3 ugrid((F + 255) / 256, (F + 7) / 8);
  for (int j = 0; j < F; ++j) {
    B200_CUDA(launch_kernel(fid_chol_pivot_kernel, dim3(1), dim3(kRed), 0, stream, (const double*)w.W, F, j, w.st,
                            w.chosen));
    B200_CUDA(launch_kernel(fid_chol_update_kernel, ugrid, dim3(256), 0, stream, w.W, w.G, F, j,
                            (const State*)w.st, (const int32_t*)w.chosen));
  }
  B200_LAUNCH_CHECK("fid_chol_update_kernel");

  // 2. T = sigma_x G (into W), M = G^T T (lower tiles, mirrored)
  GemmArgs g = {};
  g.a = {p->sigma_x, B200_DT_F64, 0, F, 1, nullptr};
  g.b = {w.G, B200_DT_F64, 0, F, 1, nullptr};
  g.M = g.N = F;
  g.K = F;
  g.alpha = 1.0;
  g.c = w.W;
  g.ldc = F;
  g.sym = 0;
  B200_CUDA(dgemm(g, stream));
  g.a = {w.G, B200_DT_F64, 1, 1, F, nullptr};
  g.b = {w.W, B200_DT_F64, 0, F, 1, nullptr};
  g.c = w.M;
  g.sym = 1;
  B200_CUDA(dgemm(g, stream));
  B200_LAUNCH_CHECK("fid_dgemm_kernel");

  // 3. tridiagonalise M in place, then bisect
  for (int k = 0; k + 2 < F; ++k) {
    const int m = F - k - 1;
    B200_CUDA(launch_kernel(fid_house_kernel, dim3(1), dim3(kRed), 0, stream, (const double*)w.M, F, k, w.d, w.e, w.v,
                            w.st));
    B200_CUDA(launch_kernel(fid_symv_kernel, dim3((m + 7) / 8), dim3(256), 0, stream, (const double*)w.M, F, k,
                            (const double*)w.v, w.pw, (const State*)w.st));
    B200_CUDA(launch_kernel(fid_house_w_kernel, dim3(1), dim3(kRed), 0, stream, F, k, (const double*)w.v, w.pw,
                            (const State*)w.st));
    B200_CUDA(launch_kernel(fid_rank2_kernel, dim3((m + 255) / 256, (m + 7) / 8), dim3(256), 0, stream, w.M, F, k,
                            (const double*)w.v, (const double*)w.pw));
  }
  B200_LAUNCH_CHECK("fid_rank2_kernel");
  B200_CUDA(launch_kernel(fid_tri_tail_kernel, dim3(1), dim3(kRed), 0, stream, (const double*)w.M, F, w.d, w.e, w.st));
  B200_LAUNCH_CHECK("fid_tri_tail_kernel");
  B200_CUDA(launch_kernel(fid_bisect_kernel, dim3((F + 127) / 128), dim3(128), 0, stream, (const double*)w.d,
                          (const double*)w.e, F, (const State*)w.st, w.eig));
  B200_LAUNCH_CHECK("fid_bisect_kernel");

  // 4. the distance
  B200_CUDA(launch_kernel(fid_finish_kernel, dim3(1), dim3(kRed), 0, stream, p->mu_x, p->sigma_x, p->mu_y, p->sigma_y,
                          F, (const double*)w.eig, (const State*)w.st, p->out, p->rank));
  B200_LAUNCH_CHECK("fid_finish_kernel");
  return B200_OK;
}
