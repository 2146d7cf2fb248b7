// fp32 parameter -> K-major h16 weight matrix for b200_igemm, one launch per weight (include/b200gen.h,
// b200_repack_weight).  Replaces the Python loops of ATen slices / adds / cats / casts that packed weights in round 1
// (~640 extra ATen launches on the first forward of the 3-D UNet).  One thread writes 8 consecutive columns of one row
// (one 16-byte store); reads of the source are strided by `taps` (the parameter is tap-minor) — a one-time pass over
// a tensor of a few MB, so coalescing of the reads is not worth a staging buffer.
#include "common.cuh"

namespace b200 {

struct RepackDev {
  const float* src;
  h16* dst;
  int cout, cin, taps, transposed, mode;
  int rows_pad, pitch, n_blocks;
  b200_repack_block blk[B200_IGEMM_MAX_SEG];
};

__device__ __forceinline__ float src_at(const RepackDev& p, int co, int c, int tap) {
  const long long idx = p.transposed ? ((long long)c * p.cout + co) * p.taps + tap
                                     : ((long long)co * p.cin + c) * p.taps + tap;
  return __ldg(p.src + idx);
}

__global__ void __launch_bounds__(256) repack_kernel(const __grid_constant__ RepackDev p) {
  const int groups = p.pitch >> 3;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)p.rows_pad * groups) return;
  const int row = (int)(idx / groups);
  const int col0 = (int)(idx % groups) * 8;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
  if (p.mode == B200_REPACK_TAP_IN) {
    if (row < p.cout) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = col0 + j;
        if (col < p.taps * p.cin) v[j] = src_at(p, row, col % p.cin, col / p.cin);
      }
    }
  } else if (p.mode == B200_REPACK_TAP_OUT) {
    if (row < p.taps * p.cout) {
      const int tap = row / p.cout, co = row % p.cout;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (col0 + j < p.cin) v[j] = src_at(p, co, col0 + j, tap);
    }
  } else if (row < p.cout) {
    // the block that owns these 8 columns (block widths are multiples of 64, so a group never straddles two)
    int b = -1;
    for (int i = 0; i < p.n_blocks; ++i) {
      const int w = ((p.blk[i].cs + 63) >> 6) << 6;
      if (col0 >= p.blk[i].col0 && col0 < p.blk[i].col0 + w) { b = i; break; }
    }
    if (b >= 0) {
      const b200_repack_block& k = p.blk[b];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = col0 + j - k.col0;
        if (c < k.cs) {
          float s = 0.f;
          for (int t = 0; t < k.ntaps; ++t) s += src_at(p, row, k.cin0 + c, k.tap[t]);   // index order, fp32
          v[j] = s;
        }
      }
    }
  }
  *reinterpret_cast<uint4*>(p.dst + (long long)row * p.pitch + col0) = pack8(v);
}

// eval-mode BatchNorm folded into the convolution before it: s = gamma / sqrt(var + eps), w' = w * s[co],
// b' = beta + (b - mean) * s.  fp64 arithmetic, one rounding to fp32 per output.
__device__ __forceinline__ double bn_scale(const float* gamma, const float* var, float eps, int co) {
  return (double)__ldg(gamma + co) / sqrt((double)__ldg(var + co) + (double)eps);
}

__global__ void __launch_bounds__(256) batchnorm_fold_kernel(const float* __restrict__ w, const float* __restrict__ b,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta,
                                                             const float* __restrict__ mean,
                                                             const float* __restrict__ var, float eps, int cout,
                                                             long long per_out, float* __restrict__ w_out,
                                                             float* __restrict__ b_out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long i = i0; i < (long long)cout * per_out; i += stride)
    w_out[i] = (float)((double)__ldg(w + i) * bn_scale(gamma, var, eps, (int)(i / per_out)));
  for (long long co = i0; co < cout; co += stride) {
    const double bias = b ? (double)__ldg(b + co) : 0.0;
    b_out[co] = (float)((double)__ldg(beta + co) + (bias - (double)__ldg(mean + co)) * bn_scale(gamma, var, eps, (int)co));
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_repack_weight(const float* src, int32_t cout, int32_t cin, int32_t taps, int32_t transposed,
                                  int32_t mode, const b200_repack_block* blocks, int32_t n_blocks, void* dst,
                                  int32_t rows_pad, int32_t dst_pitch, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(src && dst, "repack_weight: null pointer");
  B200_CHECK_ARG(cout >= 1 && cin >= 1 && taps >= 1, "repack_weight: bad weight extent %d x %d x %d", cout, cin, taps);
  B200_CHECK_ARG(dst_pitch >= 8 && dst_pitch % 8 == 0 && rows_pad >= 1 && ((uintptr_t)dst & 15) == 0,
                 "repack_weight: destination pitch must be a multiple of 8 and the pointer 16-byte aligned");
  B200_CHECK_ARG(mode >= B200_REPACK_BLOCKS && mode <= B200_REPACK_TAP_OUT, "repack_weight: unknown mode %d", mode);
  RepackDev d;
  d.src = src; d.dst = reinterpret_cast<h16*>(dst);
  d.cout = cout; d.cin = cin; d.taps = taps; d.transposed = transposed ? 1 : 0; d.mode = mode;
  d.rows_pad = rows_pad; d.pitch = dst_pitch; d.n_blocks = 0;
  if (mode == B200_REPACK_BLOCKS) {
    B200_CHECK_ARG(blocks && n_blocks >= 1 && n_blocks <= B200_IGEMM_MAX_SEG, "repack_weight: n_blocks=%d out of range",
                   n_blocks);
    B200_CHECK_ARG(rows_pad >= cout, "repack_weight: rows_pad %d < cout %d", rows_pad, cout);
    for (int i = 0; i < n_blocks; ++i) {
      const b200_repack_block& b = blocks[i];
      B200_CHECK_ARG(b.col0 >= 0 && b.col0 % 64 == 0 && b.cs >= 1 && b.cin0 >= 0 && b.cin0 + b.cs <= cin &&
                     b.col0 + ((b.cs + 63) / 64) * 64 <= dst_pitch && b.ntaps >= 1 && b.ntaps <= 8,
                     "repack_weight: block %d invalid (col0 %d, cin0 %d, cs %d, ntaps %d)", i, b.col0, b.cin0, b.cs, b.ntaps);
      for (int t = 0; t < b.ntaps; ++t)
        B200_CHECK_ARG(b.tap[t] >= 0 && b.tap[t] < taps, "repack_weight: block %d tap %d out of range", i, b.tap[t]);
      d.blk[i] = b;
    }
    d.n_blocks = n_blocks;
  } else if (mode == B200_REPACK_TAP_IN) {
    B200_CHECK_ARG(!transposed && taps * cin <= dst_pitch && rows_pad >= cout, "repack_weight(tap_in): extents");
  } else {
    B200_CHECK_ARG(!transposed && cin <= dst_pitch && rows_pad >= taps * cout, "repack_weight(tap_out): extents");
  }
  const long long total = (long long)rows_pad * (dst_pitch / 8);
  B200_CHECK_ARG((total + 255) / 256 < (1ll << 31), "repack_weight: weight too large");
  B200_CUDA(b200::launch_kernel(repack_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, d));
  B200_LAUNCH_CHECK("repack_kernel");
  return B200_OK;
}

extern "C" int b200_batchnorm_fold(const float* w, const float* b, const float* gamma, const float* beta,
                                   const float* mean, const float* var, float eps, int32_t cout, int64_t per_out,
                                   float* w_out, float* b_out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(w && gamma && beta && mean && var && w_out && b_out, "batchnorm_fold: null pointer");
  B200_CHECK_ARG(cout >= 1 && per_out >= 1 && eps >= 0.f, "batchnorm_fold: bad extent %d x %lld or eps", cout,
                 (long long)per_out);
  const long long blocks = ((long long)cout * per_out + 255) / 256;
  B200_CHECK_ARG(blocks < (1ll << 31), "batchnorm_fold: weight too large");
  B200_CUDA(b200::launch_kernel(batchnorm_fold_kernel, (unsigned)blocks, 256, 0, stream, w, b, gamma, beta, mean, var, eps,
                             (int)cout, (long long)per_out, w_out, b_out));
  B200_LAUNCH_CHECK("batchnorm_fold_kernel");
  return B200_OK;
}
