// Implicit-GEMM convolution / GEMM on Hopper wgmma tensor cores.
//
// Replaces every dense contraction of the reference sampling path (the cuDNN / cuBLAS calls behind
// monai Convolution, nn.Linear, torch.baddbmm/bmm — see include/b200gen.h for the call sites).
//
// Design:
//   * activations live in HBM as channels-last 16-bit rows; a CTA tile is a BW x BH x BD box of 128 output
//     voxels x BN output channels.  For every filter tap and every 64-channel chunk the producer
//     thread issues ONE tiled-TMA box load of the shifted input box: out-of-range coordinates
//     (the zero padding, ragged edges, channel tails) are zero-filled by the TMA unit, stride-2
//     convolutions use the tensor map's traversal stride.  No im2col buffer ever exists.
//   * the box lands in shared memory as a 128-row x 128-byte SWIZZLE_128B K-major tile — the canonical
//     wgmma operand layout — and two warpgroups issue wgmma (M=64 each, N=BN, K=16) accumulating in
//     registers.  Weights are a K-major [Cout][taps*Cin] 16-bit matrix, also TMA-staged.
//   * warp-specialised persistent kernel: 4 epilogue warps, 2 MMA warpgroups, 1 TMA producer warp; smem ring of
//     STAGES {A,B} tiles (full/empty mbarriers); the finished accumulator goes through one fp32 shared-memory tile so
//     the epilogue of tile i overlaps the main loop of tile i+1.
//   * fused epilogue: +bias, +per-sample row vector (time embedding), activation, scale, +residual, activation,
//     16-bit/fp32 store with arbitrary voxel strides (so transposed-conv phases and channel-slice outputs need no
//     extra pass).
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <mutex>
#include <string.h>

namespace b200 {

static constexpr int kBM = 128;           // rows (output voxels) per tile: two wgmma M=64 warpgroups
static constexpr int kBK = 64;            // channels per K chunk == 128 bytes of 16-bit data == swizzle span
static constexpr int kABytes = kBM * kBK * 2;
static constexpr int kMmaWarp0 = 4;       // warps 0..3 epilogue, 4..11 two MMA warpgroups, 12 TMA producer
static constexpr int kTmaWarp = 12;
static constexpr int kThreads = 13 * 32;

struct SegDev {
  int8_t src, dw, dh, dd;
  uint16_t c0, nchunks;
};

struct IgemmDev {
  alignas(64) CUtensorMap tmA[2];
  alignas(64) CUtensorMap tmB;
  // raw views for the cross-check kernel
  const h16* a_ptr[2];
  int a_C[2], a_pitch[2];
  int in_N, in_D, in_H, in_W;
  int a_bcast;              // 1: every sample reads A at batch index 0
  const h16* w_ptr;
  int w_rows, w_K, w_pitch;
  long long w_bstride;
  int w_batched;
  // geometry
  int n_seg, num_k_chunks;
  int sd, sh, sw;
  int N, OD, OH, OW;
  int BW, BH, BD, bw_log2, bh_log2;
  int tiles_w, tiles_h, tiles_d, tiles_n, num_tiles;
  int k_splits;             // >= 1: the reduction of every tile is cut into this many chunk ranges (fastest tile index)
  long long split_stride;   // output elements between the partial results of consecutive ranges
  // epilogue
  void* out_ptr;
  int out_dtype, cout, out_cols, out_vec, out_staged, out_v256;
  float* stat_ptr;          // optional [rows][tiles_n][2] (max, sum exp) per row and column tile
  float* gn_partial;        // optional [N][gn_slots][cout/8][2] (sum, sum of squares) of the bf16 outputs, 8-channel groups
  int gn_slots, gn_slot0;
  int gn_sh;                // log2 of the channels per partial group: 3 (8 channels) or 2 (4 channels)
  long long out_sN, out_sD, out_sH, out_sW;
  const float* bias;
  const float* rowvec;
  long long rowvec_bstride;
  const float* row_bias;
  int act1, act2;
  int geglu;                // act1 was B200_ACT_GEGLU: [32 a | 32 gate] column groups -> a * gelu(gate), cout / 2 output channels
  float scale;
  const void* res_ptr;
  int res_dtype, res_vec, res_v256;
  long long res_sN, res_sD, res_sH, res_sW;
  SegDev seg[B200_IGEMM_MAX_SEG];
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* tm, uint32_t bar, uint32_t dst, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// CH consecutive fp32 accumulator values of one tile row from the shared-memory hand-off tile
template <int CH>
__device__ __forceinline__ void acc_ld(const float* src, uint32_t* r) {
#pragma unroll
  for (int j = 0; j < CH; j += 4) {
    const float4 t = *reinterpret_cast<const float4*>(src + j);
    r[j] = __float_as_uint(t.x); r[j + 1] = __float_as_uint(t.y);
    r[j + 2] = __float_as_uint(t.z); r[j + 3] = __float_as_uint(t.w);
  }
}

// first reduction chunk of range `ks` when `num_k` chunks are cut into `splits` near-equal ranges
__host__ __device__ __forceinline__ int split_begin(int num_k, int splits, int ks) {
  return (int)(((long long)num_k * ks) / splits);
}

// ------------------------------------------------------------------------------------------------
// Fused epilogue for CH consecutive columns of one output row (shared by both kernels).
// ------------------------------------------------------------------------------------------------
template <int CH>
__device__ __forceinline__ void epilogue_math(const IgemmDev& p, float* v, int nb, int ow, long long res_off,
                                              int col0) {
  // bias + per-sample row vector (+ per-row bias for transposed-operand GEMMs)
  const float rb = p.row_bias ? __ldg(p.row_bias + ow) : 0.f;
#pragma unroll
  for (int j = 0; j < CH; ++j) {
    int col = col0 + j;
    float add = rb;
    if (col < p.cout) {
      if (p.bias) add += __ldg(p.bias + col);
      if (p.rowvec) add += __ldg(p.rowvec + (long long)nb * p.rowvec_bstride + col);
    }
    float x = v[j] + add;
    x = apply_act(x, p.act1);
    v[j] = x * p.scale;
  }
  if (p.res_ptr) {
    if (p.res_dtype == B200_DT_H16) {
      const h16* r = reinterpret_cast<const h16*>(p.res_ptr) + res_off + col0;
      if (p.res_vec) {
#pragma unroll
        for (int g = 0; g < CH / 8; ++g) {
          if (col0 + g * 8 < p.out_cols) {
            uint4 t = __ldg(reinterpret_cast<const uint4*>(r + g * 8));
            float f[8];
            unpack8(t, f);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[g * 8 + j] += f[j];
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < CH; ++j)
          if (col0 + j < p.out_cols) v[j] += h2f(r[j]);
      }
    } else {
      const float* r = reinterpret_cast<const float*>(p.res_ptr) + res_off + col0;
      if (p.res_vec) {
#pragma unroll
        for (int g = 0; g < CH / 4; ++g) {
          if (col0 + g * 4 < p.out_cols) {
            float4 t = __ldg(reinterpret_cast<const float4*>(r + g * 4));
            v[g * 4 + 0] += t.x; v[g * 4 + 1] += t.y; v[g * 4 + 2] += t.z; v[g * 4 + 3] += t.w;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < CH; ++j)
          if (col0 + j < p.out_cols) v[j] += r[j];
      }
    }
  }
  if (p.act2 != B200_ACT_NONE) {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = apply_act(v[j], p.act2);
  }
  // columns in [cout, out_cols) are padding: force exact zeros
#pragma unroll
  for (int j = 0; j < CH; ++j)
    if (col0 + j >= p.cout) v[j] = 0.f;
}

// each thread stores its own row segment (good when consecutive rows are adjacent in memory: conv outputs)
template <int CH>
__device__ __forceinline__ void store_direct(const IgemmDev& p, const float* v, long long out_off, int col0) {
  if (p.out_dtype == B200_DT_H16) {
    h16* o = reinterpret_cast<h16*>(p.out_ptr) + out_off + col0;
    if (p.out_vec) {
#pragma unroll
      for (int g = 0; g < CH / 8; ++g)
        if (col0 + g * 8 < p.out_cols) *reinterpret_cast<uint4*>(o + g * 8) = pack8(v + g * 8);
    } else {
#pragma unroll
      for (int j = 0; j < CH; ++j)
        if (col0 + j < p.out_cols) o[j] = f2h(v[j]);
    }
  } else {
    float* o = reinterpret_cast<float*>(p.out_ptr) + out_off + col0;
    if (p.out_vec) {
#pragma unroll
      for (int g = 0; g < CH / 4; ++g)
        if (col0 + g * 4 < p.out_cols)
          *reinterpret_cast<float4*>(o + g * 4) =
              make_float4(v[g * 4], v[g * 4 + 1], v[g * 4 + 2], v[g * 4 + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < CH; ++j)
        if (col0 + j < p.out_cols) o[j] = v[j];
    }
  }
}


// ------------------------------------------------------------------------------------------------
// Fast epilogue (full CH-column chunks of vector-aligned outputs): the general path above re-derives bias / row-vector
// addresses, activation switches and bounds per ELEMENT (~55 instructions per output value — with one epilogue warp
// per scheduler that made the epilogue, not the tensor pipe, the critical path of every K <= 7k convolution).  Here
// the additive vector comes from shared memory (filled once per (sample, column tile)), the activation switches are
// hoisted out of the element loops and the residual / output move as 256-bit (or 128-bit) vectors.
// ------------------------------------------------------------------------------------------------
// 32 bytes as two 16-byte accesses (sm_90 has no 256-bit global load / store)
__device__ __forceinline__ void ldg256(const void* ptr, uint4& a, uint4& b) {
  a = __ldg(reinterpret_cast<const uint4*>(ptr));
  b = __ldg(reinterpret_cast<const uint4*>(ptr) + 1);
}
__device__ __forceinline__ void stg256(void* ptr, const uint4& a, const uint4& b) {
  reinterpret_cast<uint4*>(ptr)[0] = a;
  reinterpret_cast<uint4*>(ptr)[1] = b;
}
template <int CH>
__device__ __forceinline__ void act_inplace(float* v, int act) {
  if (act == B200_ACT_NONE) return;
  if (act == B200_ACT_SILU) {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = silu_f(v[j]);
  } else if (act == B200_ACT_LEAKYRELU || act == B200_ACT_LEAKYRELU02) {
    const float slope = act == B200_ACT_LEAKYRELU ? 0.01f : 0.2f;
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = v[j] > 0.0f ? v[j] : slope * v[j];
  } else if (act == B200_ACT_GELU) {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = 0.5f * v[j] * (1.0f + erff(v[j] * 0.70710678118654752f));
  } else if (act == B200_ACT_TANH || act == B200_ACT_SIGMOID) {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = apply_act(v[j], act);
  } else {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = fmaxf(v[j], 0.0f);
  }
}
// residual prefetch for one row chunk (bf16, 16-byte aligned): CH/8 uint4
template <int CH>
__device__ __forceinline__ void load_res_fast(const IgemmDev& p, uint4* rv, long long res_off, int col0) {
  const h16* r = reinterpret_cast<const h16*>(p.res_ptr) + res_off + col0;
  if (p.res_v256) {
#pragma unroll
    for (int g = 0; g < CH / 16; ++g) ldg256(r + g * 16, rv[2 * g], rv[2 * g + 1]);
  } else {
#pragma unroll
    for (int g = 0; g < CH / 8; ++g) rv[g] = __ldg(reinterpret_cast<const uint4*>(r + g * 8));
  }
}
template <int CH>
__device__ __forceinline__ void epilogue_fast(const IgemmDev& p, const uint32_t* raw, const float* addv,
                                              const uint4* rv, long long out_off, int col0, float* gs) {
  float v[CH];
#pragma unroll
  for (int j = 0; j < CH; j += 4) {
    const float4 a = *reinterpret_cast<const float4*>(addv + j);
    v[j] = __uint_as_float(raw[j]) + a.x;
    v[j + 1] = __uint_as_float(raw[j + 1]) + a.y;
    v[j + 2] = __uint_as_float(raw[j + 2]) + a.z;
    v[j + 3] = __uint_as_float(raw[j + 3]) + a.w;
  }
  act_inplace<CH>(v, p.act1);
  if (p.scale != 1.0f) {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] *= p.scale;
  }
  if (p.res_ptr) {
#pragma unroll
    for (int g = 0; g < CH / 8; ++g) {
      float f[8];
      unpack8(rv[g], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[g * 8 + j] += f[j];
    }
  }
  act_inplace<CH>(v, p.act2);
  if (p.out_dtype == B200_DT_H16) {
    h16* o = reinterpret_cast<h16*>(p.out_ptr) + out_off + col0;
    uint4 pk[CH / 8];
#pragma unroll
    for (int g = 0; g < CH / 8; ++g) pk[g] = pack8(v + g * 8);
    if (p.out_v256) {
#pragma unroll
      for (int g = 0; g < CH / 16; ++g) stg256(o + g * 16, pk[2 * g], pk[2 * g + 1]);
    } else {
#pragma unroll
      for (int g = 0; g < CH / 8; ++g) *reinterpret_cast<uint4*>(o + g * 8) = pk[g];
    }
    if (gs) {   // GroupNorm partials of the values as stored (16-bit-rounded)
      constexpr int G8 = CH / 8, G4 = CH / 4;
      if (p.gn_sh == 3) {          // one 8-channel group per 16-byte vector: gs[0, G8) sums, gs[G8, 2 G8) sums of squares
#pragma unroll
        for (int g = 0; g < G8; ++g) {
          float f[8];
          unpack8(pk[g], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) { gs[g] += f[j]; gs[G8 + g] = fmaf(f[j], f[j], gs[G8 + g]); }
        }
      } else {                     // 4-channel groups (GroupNorm(32) over 128 channels): gs[0, G4) sums, gs[G4, 2 G4) squares
#pragma unroll
        for (int g = 0; g < G8; ++g) {
          float f[8];
          unpack8(pk[g], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            gs[2 * g + (j >> 2)] += f[j];
            gs[G4 + 2 * g + (j >> 2)] = fmaf(f[j], f[j], gs[G4 + 2 * g + (j >> 2)]);
          }
        }
      }
    }
  } else {
    float* o = reinterpret_cast<float*>(p.out_ptr) + out_off + col0;
#pragma unroll
    for (int g = 0; g < CH / 4; ++g)
      *reinterpret_cast<float4*>(o + g * 4) = make_float4(v[g * 4], v[g * 4 + 1], v[g * 4 + 2], v[g * 4 + 3]);
  }
}

template <int CH>
__device__ __forceinline__ void epilogue_row(const IgemmDev& p, float* v, int nb, int ow, long long out_off,
                                             long long res_off, int col0) {
  epilogue_math<CH>(p, v, nb, ow, res_off, col0);
  store_direct<CH>(p, v, out_off, col0);
}

// The leanest epilogue: out = h16(acc + bias/row-vector [+ residual]) for a full CH-column chunk of a 32-byte-aligned h16
// output — every nn.Linear of the transformer blocks, 1x1 projections.  Same arithmetic and order as epilogue_fast
// with act1 = act2 = none and scale = 1 (bit-identical), but none of its run-time switches: with one epilogue warp per
// scheduler the ~20 uniform branches per chunk of the general body (activation chains, scale, output type, statistics)
// and its instruction footprint, not the tensor cores, bound a GEMM with a short (K = 256) reduction.
template <int CH, bool HAS_RES>
__device__ __forceinline__ void epilogue_lean(const IgemmDev& p, const uint32_t* raw, const float* addv,
                                              const uint4* rv, long long out_off, int col0) {
  float v[CH];
#pragma unroll
  for (int j = 0; j < CH; j += 4) {
    const float4 a = *reinterpret_cast<const float4*>(addv + j);
    v[j] = __uint_as_float(raw[j]) + a.x;
    v[j + 1] = __uint_as_float(raw[j + 1]) + a.y;
    v[j + 2] = __uint_as_float(raw[j + 2]) + a.z;
    v[j + 3] = __uint_as_float(raw[j + 3]) + a.w;
  }
  if constexpr (HAS_RES) {
#pragma unroll
    for (int g = 0; g < CH / 8; ++g) {
      float f[8];
      unpack8(rv[g], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[g * 8 + j] += f[j];
    }
  }
  h16* o = reinterpret_cast<h16*>(p.out_ptr) + out_off + col0;
  uint4 pk[CH / 8];
#pragma unroll
  for (int g = 0; g < CH / 8; ++g) pk[g] = pack8(v + g * 8);
  if (p.out_v256) {
#pragma unroll
    for (int g = 0; g < CH / 16; ++g) stg256(o + g * 16, pk[2 * g], pk[2 * g + 1]);
  } else {
#pragma unroll
    for (int g = 0; g < CH / 8; ++g) *reinterpret_cast<uint4*>(o + g * 8) = pk[g];
  }
}

// Row-coalesced store for wide row-major outputs (GEMM-shaped calls whose rows are far apart in memory, e.g. the
// 89 600-column attention score matrix): the warp's 32 x CH tile goes through a padded shared-memory tile so that
// every store instruction writes one contiguous CH-element row segment instead of 32 scattered 16-byte pieces.
template <int CH>
__device__ __forceinline__ void store_staged(const IgemmDev& p, const float* v, float* tile /*[32][CH+1]*/,
                                             bool row_ok, long long out_off, int col0, int lane) {
  constexpr int LD = CH + 1;
#pragma unroll
  for (int j = 0; j < CH; ++j) tile[lane * LD + j] = v[j];
  __syncwarp();
  const unsigned okmask = __ballot_sync(0xffffffffu, row_ok);
  const int col = col0 + (lane % CH);
  const bool col_ok = col < p.out_cols;
  constexpr int ROWS_PER_IT = 32 / CH;      // CH == 32 -> 1 row per instruction, CH == 16 -> 2 rows
#pragma unroll 4
  for (int rr = 0; rr < 32; rr += ROWS_PER_IT) {
    const int r = rr + lane / CH;
    const long long off = __shfl_sync(0xffffffffu, out_off, r);
    if (((okmask >> r) & 1u) && col_ok) {
      const float x = tile[r * LD + (lane % CH)];
      if (p.out_dtype == B200_DT_H16)
        reinterpret_cast<h16*>(p.out_ptr)[off + col] = f2h(x);
      else
        reinterpret_cast<float*>(p.out_ptr)[off + col] = x;
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// The wgmma kernel
// ------------------------------------------------------------------------------------------------
// Warp roles (416 threads): warps 0..3 = epilogue (thread <-> tile row), warps 4..11 = two MMA warpgroups (rows 0..63
// and 64..127 of the tile), warp 12 = TMA producer.  The MMA warpgroups hold the accumulator of the tile in flight in
// registers and hand the finished tile to the epilogue through one fp32 shared-memory buffer, so the epilogue of tile i
// overlaps the main loop of tile i + 1.
template <int BN, int STAGES>
__global__ void __launch_bounds__(kThreads, 1) igemm_tc_kernel(const __grid_constant__ IgemmDev p) {
  constexpr int kBBytes = BN * kBK * 2;
  constexpr int kStageBytes = kABytes + kBBytes;
  constexpr int kAccLd = BN + 4;          // padded fp32 row: row-per-thread 16-byte reads are conflict-free
  constexpr int CH = (BN >= 32) ? 32 : 16;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + STAGES * kStageBytes;
  float* acc_smem = reinterpret_cast<float*>(smem_raw + (acc_base - smem_u32(smem_raw)));      // [kBM][kAccLd]
  const uint32_t bar_base = acc_base + kBM * kAccLd * 4;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t tfull_bar = bar_base + 8u * (2 * STAGES);
  const uint32_t tempty_bar = bar_base + 8u * (2 * STAGES + 1);
  float* stage_tiles = reinterpret_cast<float*>(smem_raw + (bar_base + 256u - smem_u32(smem_raw)));   // 4 x [32][CH+1]
  float* add_tiles = stage_tiles + 4 * 32 * 33;                                                      // 4 x 2 x [BN]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int worker = (int)blockIdx.x;
  const int n_workers = (int)gridDim.x;

  if (warp == kTmaWarp && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);          // one arrival per MMA warp
    }
    mbar_init(tfull_bar, 8);
    mbar_init(tempty_bar, 4);              // one arrival per epilogue warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  const int num_k = p.num_k_chunks;
  // work-unit index -> (k-split, column tile, spatial tile, sample)
  struct TileIdx { int ks, nt, wt, ht, dt, nb; };
  auto decode_tile = [&](int tile) {
    TileIdx t;
    int x = tile;
    t.ks = x % p.k_splits; x /= p.k_splits;
    t.nt = x % p.tiles_n; x /= p.tiles_n;
    t.wt = x % p.tiles_w; x /= p.tiles_w;
    t.ht = x % p.tiles_h; x /= p.tiles_h;
    t.dt = x % p.tiles_d; x /= p.tiles_d;
    t.nb = x;
    return t;
  };

  if (warp == kTmaWarp) {
    // ============================== TMA producer ==============================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = worker; tile < p.num_tiles; tile += n_workers) {
        const TileIdx ti = decode_tile(tile);
        const int ks = ti.ks, nt = ti.nt, wt = ti.wt, ht = ti.ht, dt = ti.dt, nb = ti.nb;
        const int iw0 = wt * p.BW * p.sw, ih0 = ht * p.BH * p.sh, id0 = dt * p.BD * p.sd;
        const int n0 = nt * BN;
        const int wb = p.w_batched ? nb : 0;
        const int a_nb = p.a_bcast ? 0 : nb;
        const int k_begin = split_begin(num_k, p.k_splits, ks), k_end = split_begin(num_k, p.k_splits, ks + 1);
        int kglob = 0;
        for (int s = 0; s < p.n_seg; ++s) {
          const SegDev sg = p.seg[s];
          if (kglob + sg.nchunks <= k_begin || kglob >= k_end) { kglob += sg.nchunks; continue; }
          const CUtensorMap* tm = &p.tmA[sg.src];
          const int cw = iw0 + sg.dw, ch = ih0 + sg.dh, cd = id0 + sg.dd;
          for (int c = 0; c < sg.nchunks; ++c, ++kglob) {
            if (kglob < k_begin || kglob >= k_end) continue;
            mbar_wait(empty_bar(stage), phase ^ 1u);
            const uint32_t a_dst = smem_base + stage * kStageBytes;
            mbar_arrive_expect_tx(full_bar(stage), kStageBytes);
            tma_load_5d(tm, full_bar(stage), a_dst, (sg.c0 + c) * kBK, cw, ch, cd, a_nb);
            tma_load_3d(&p.tmB, full_bar(stage), a_dst + kABytes, kglob * kBK, n0, wb);
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else if (warp >= kMmaWarp0) {
    // ============================== MMA warpgroups ==============================
    const int wg = (warp - kMmaWarp0) >> 2;       // rows 64 * wg .. 64 * wg + 63 of the tile
    const int wq = (warp - kMmaWarp0) & 3;        // 16-row slice of those inside the warpgroup
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = worker; tile < p.num_tiles; tile += n_workers, ++it) {
      const int ks = tile % p.k_splits;
      const int nk = split_begin(num_k, p.k_splits, ks + 1) - split_begin(num_k, p.k_splits, ks);
      int prev = -1;
      for (int k = 0; k < nk; ++k) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t a_addr = smem_base + stage * kStageBytes + wg * (64 * kBK * 2);
        const uint64_t adesc = wgmma_desc(a_addr);
        const uint64_t bdesc = wgmma_desc(smem_base + stage * kStageBytes + kABytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBK / 16; ++kk)
          wgmma_ss<BN>(acc, adesc + 2u * kk, bdesc + 2u * kk, (k | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();            // the group of the previous chunk has finished reading its stage
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(prev));
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_touch<BN / 2>(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      // hand the tile to the epilogue once it has finished reading the previous one
      mbar_wait(tempty_bar, (it & 1) ^ 1u);
      const int r0 = wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        *reinterpret_cast<float2*>(acc_smem + r0 * kAccLd + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(acc_smem + (r0 + 8) * kAccLd + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(tfull_bar);
    }
  } else {
    // ============================== epilogue warps ==============================
    const int r = warp * 32 + lane;         // row of the tile
    const float* acc_row = acc_smem + r * kAccLd;
    const int rw = r & (p.BW - 1);
    const int rh = (r >> p.bw_log2) & (p.BH - 1);
    const int rd = r >> (p.bw_log2 + p.bh_log2);
    float* addv = add_tiles + warp * 2 * BN;      // two buffers: the current vector and the prefetched next one
    float* addv_other = addv + BN;
    int next_key = -1;
    int add_key = -1;
    const bool fast_ok = p.out_vec && !p.out_staged && !p.stat_ptr &&
                         (!p.res_ptr || (p.res_vec && p.res_dtype == B200_DT_H16));
    const bool lean_ok = fast_ok && p.act1 == B200_ACT_NONE && p.act2 == B200_ACT_NONE && p.scale == 1.0f &&
                         !p.row_bias && !p.gn_partial && p.out_dtype == B200_DT_H16 && !p.geglu;
    // GroupNorm partial sums for the consumer of this tensor: per warp [BN/8 groups][sum, sumsq] in shared memory
    // (aliases the staged-store tiles, which this mode excludes), flushed to this warp's private global slot
    // whenever the (sample, column tile) changes and at the end — deterministic, no atomics.
    float* gacc = stage_tiles + warp * (32 * 33);
    const bool gn_on = (p.gn_partial != nullptr);
    int gn_nb = -1, gn_n0 = 0;
    auto gn_flush = [&]() {
      if (gn_nb >= 0) {
        const int sh = p.gn_sh;
        float* dst = p.gn_partial +
                     (((long long)gn_nb * p.gn_slots + p.gn_slot0 + blockIdx.x * 4 + warp) * (p.cout >> sh)) * 2 +
                     (gn_n0 >> sh) * 2;
        for (int e = lane; e < (BN >> sh) * 2; e += 32) {
          if (gn_n0 + ((e >> 1) << sh) < p.cout) dst[e] += gacc[e];
        }
      }
      for (int e = lane; e < (BN >> 2) * 2; e += 32) gacc[e] = 0.f;
      __syncwarp();
    };
    if (gn_on) gn_flush();
    int it = 0;
    for (int tile = worker; tile < p.num_tiles; tile += n_workers, ++it) {
      const TileIdx ti = decode_tile(tile);
      const int ks = ti.ks, nt = ti.nt, wt = ti.wt, ht = ti.ht, dt = ti.dt;
      const int nb = ti.nb;
      const int ow = wt * p.BW + rw, oh = ht * p.BH + rh, od = dt * p.BD + rd;
      const bool row_ok = (ow < p.OW) && (oh < p.OH) && (od < p.OD);
      const int n0 = nt * BN;

      constexpr int PER = (BN + 31) / 32;
      if (fast_ok && add_key != nb * p.tiles_n + nt && next_key == nb * p.tiles_n + nt) {
        // the vector was requested during the previous tile's epilogue and sits in the other buffer
        if (gn_on) { gn_flush(); gn_nb = nb; gn_n0 = n0; }
        add_key = next_key;
        next_key = -1;
        float* t = addv; addv = addv_other; addv_other = t;
      }
      if (fast_ok && add_key != nb * p.tiles_n + nt) {
        if (gn_on) { gn_flush(); gn_nb = nb; gn_n0 = n0; }
        // bias + per-sample row vector of this (sample, column tile): shared by all rows, refreshed only on change
        add_key = nb * p.tiles_n + nt;
        __syncwarp();
        {
          // all loads first: with the column tile as the fastest tile index a GEMM-shaped call refreshes this vector
          // for EVERY tile, and a load -> add chain per element would cost eight L2 round trips per tile
          float bv[PER], rw[PER];
#pragma unroll
          for (int i = 0; i < PER; ++i) {
            const int col = n0 + lane + 32 * i;
            const bool ok = (lane + 32 * i < BN) && col < p.cout;
            bv[i] = (ok && p.bias) ? __ldg(p.bias + col) : 0.f;
            rw[i] = (ok && p.rowvec) ? __ldg(p.rowvec + (long long)nb * p.rowvec_bstride + col) : 0.f;
          }
#pragma unroll
          for (int i = 0; i < PER; ++i)
            if (lane + 32 * i < BN) addv[lane + 32 * i] = bv[i] + rw[i];
        }
        __syncwarp();
      }
      // the NEXT tile's vector, if it differs: requested now, written to the other buffer after this tile's chunks (one
      // exposed L2 round trip per tile otherwise)
      float nbv[PER], nrw[PER];
      int want_key = -1;
      if (fast_ok && tile + n_workers < p.num_tiles) {
        const TileIdx tn = decode_tile(tile + n_workers);
        if (tn.nb < p.N && tn.nb * p.tiles_n + tn.nt != add_key) {
          want_key = tn.nb * p.tiles_n + tn.nt;
#pragma unroll
          for (int i = 0; i < PER; ++i) {
            const int col = tn.nt * BN + lane + 32 * i;
            const bool ok = (lane + 32 * i < BN) && col < p.cout;
            nbv[i] = (ok && p.bias) ? __ldg(p.bias + col) : 0.f;
            nrw[i] = (ok && p.rowvec) ? __ldg(p.rowvec + (long long)tn.nb * p.rowvec_bstride + col) : 0.f;
          }
        }
      }

      // residual of the first full chunk: in flight while this warp waits for the accumulator; every later chunk's
      // residual is requested one chunk ahead (a load -> use chain per chunk exposed one HBM / L2 latency per 32
      // columns: the epilogue warps are one per scheduler, nothing else hides it)
      const long long res_off = nb * p.res_sN + od * p.res_sD + oh * p.res_sH + ow * p.res_sW;
      const bool res_fast = fast_ok && p.res_ptr && row_ok;
      uint4 rv_next[CH / 8];
      if (res_fast && n0 + CH <= p.cout) load_res_fast<CH>(p, rv_next, res_off, n0);

      mbar_wait(tfull_bar, it & 1);
      // out_off (like res_off above) is formed next to its first use: held across the wait and the vector refresh, the
      // two pushed the 32-column instantiation into per-tile spills at the 128-register cap
      const long long out_off = nb * p.out_sN + od * p.out_sD + oh * p.out_sH + ow * p.out_sW + ks * p.split_stride;
      float run_max = -INFINITY, run_sum = 0.f;
      float* my_tile = stage_tiles + warp * (32 * (CH + 1));
      int c0 = 0;
      if constexpr (CH == 32 && BN >= 64) {
        if (p.geglu) {
          // GEGLU feed-forward: this GEMM's columns are [32 a | 32 gate] groups; out = (a + b_a) * gelu(gate + b_g) on
          // the fp32 accumulators (the unfused path rounded linear1's output to 16 bits first and spent a 200 MB pass
          // per block on the gating), half as many channels stored
#pragma unroll 1
          for (; c0 + 64 <= BN && n0 + c0 + 64 <= p.cout; c0 += 64) {
            uint32_t ra[32], rg[32];
            acc_ld<32>(acc_row + c0, ra);
            acc_ld<32>(acc_row + c0 + 32, rg);
            if (row_ok) {
              float v[32];
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float4 ba = *reinterpret_cast<const float4*>(addv + c0 + j);
                const float4 bg = *reinterpret_cast<const float4*>(addv + c0 + 32 + j);
                const float a4[4] = {ba.x, ba.y, ba.z, ba.w}, g4[4] = {bg.x, bg.y, bg.z, bg.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float a = __uint_as_float(ra[j + e]) + a4[e];
                  const float g = __uint_as_float(rg[j + e]) + g4[e];
                  v[j + e] = a * (0.5f * g * (1.0f + erff(g * 0.70710678118654752f)));
                }
              }
              h16* o = reinterpret_cast<h16*>(p.out_ptr) + out_off + ((n0 + c0) >> 1);
              uint4 pk[4];
#pragma unroll
              for (int g = 0; g < 4; ++g) pk[g] = pack8(v + g * 8);
              if (p.out_v256) {
                stg256(o, pk[0], pk[1]);
                stg256(o + 16, pk[2], pk[3]);
              } else {
#pragma unroll
                for (int g = 0; g < 4; ++g) *reinterpret_cast<uint4*>(o + g * 8) = pk[g];
              }
            }
          }
          c0 = BN;       // cout is a multiple of 64: every real column of this tile has been consumed
        }
      }
      if (lean_ok) {
#pragma unroll 1
        for (; c0 < BN && n0 + c0 + CH <= p.cout; c0 += CH) {       // warp-uniform: full chunks of real columns
          uint4 rv[CH / 8];
#pragma unroll
          for (int g = 0; g < CH / 8; ++g) rv[g] = rv_next[g];
          if (res_fast && c0 + CH < BN && n0 + c0 + 2 * CH <= p.cout)
            load_res_fast<CH>(p, rv_next, res_off, n0 + c0 + CH);
          uint32_t raw[CH];
          acc_ld<CH>(acc_row + c0, raw);
          if (row_ok) {
            if (p.res_ptr) epilogue_lean<CH, true>(p, raw, addv + c0, rv, out_off, n0 + c0);
            else epilogue_lean<CH, false>(p, raw, addv + c0, rv, out_off, n0 + c0);
          }
        }
      }
#pragma unroll 1
      for (; c0 < BN; c0 += CH) {
        if (n0 + c0 >= p.out_cols) break;             // warp-uniform
        if (fast_ok && n0 + c0 + CH <= p.cout) {      // warp-uniform: a full chunk of real columns
          uint4 rv[CH / 8];
#pragma unroll
          for (int g = 0; g < CH / 8; ++g) rv[g] = rv_next[g];
          if (res_fast && c0 + CH < BN && n0 + c0 + 2 * CH <= p.cout)
            load_res_fast<CH>(p, rv_next, res_off, n0 + c0 + CH);      // next chunk's residual, one chunk ahead
          uint32_t raw[CH];
          acc_ld<CH>(acc_row + c0, raw);
          float gs[16] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (row_ok) {
            if (p.row_bias) {                       // operand-swapped GEMMs (V^T = W X^T): the bias runs along the rows
              const float rb = __ldg(p.row_bias + ow);
#pragma unroll
              for (int j = 0; j < CH; ++j) raw[j] = __float_as_uint(__uint_as_float(raw[j]) + rb);
            }
            epilogue_fast<CH>(p, raw, addv + c0, rv, out_off, n0 + c0, gn_on ? gs : nullptr);
          }
          if constexpr (CH == 32) {
            if (gn_on && p.gn_sh == 2) {
              // 16 values x 32 lanes -> one total per lane: transpose-reduce over lane bits 4,3,2,1, butterfly over 0;
              // the lane then holds statistic (lane >> 4) of 4-channel group 4 * bit3 + 2 * bit2 + bit1 of this chunk
              float a8[8], a4[4], a2[2];
              bool hi = (lane & 16) != 0;
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float send = hi ? gs[i] : gs[8 + i], keep = hi ? gs[8 + i] : gs[i];
                a8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
              }
              hi = (lane & 8) != 0;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float send = hi ? a8[i] : a8[4 + i], keep = hi ? a8[4 + i] : a8[i];
                a4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
              }
              hi = (lane & 4) != 0;
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const float send = hi ? a4[i] : a4[2 + i], keep = hi ? a4[2 + i] : a4[i];
                a2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
              }
              hi = (lane & 2) != 0;
              float c = (hi ? a2[1] : a2[0]) + __shfl_xor_sync(0xffffffffu, hi ? a2[0] : a2[1], 2);
              c += __shfl_xor_sync(0xffffffffu, c, 1);
              if ((lane & 1) == 0) {
                const int grp = (c0 >> 2) + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
                gacc[grp * 2 + (lane >> 4)] += c;
              }
            } else if (gn_on) {
              // 8 values x 32 lanes -> one total per lane: transpose-reduce over lane bits 4,3,2, butterfly over 1,0;
              // the lane then holds statistic (lane >> 4) of group 2 * bit3 + bit2 of this 32-column chunk
              float a[4], b[2];
              bool hi = (lane & 16) != 0;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float send = hi ? gs[i] : gs[4 + i], keep = hi ? gs[4 + i] : gs[i];
                a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
              }
              hi = (lane & 8) != 0;
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const float send = hi ? a[i] : a[2 + i], keep = hi ? a[2 + i] : a[i];
                b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
              }
              hi = (lane & 4) != 0;
              float c = (hi ? b[1] : b[0]) + __shfl_xor_sync(0xffffffffu, hi ? b[0] : b[1], 4);
              c += __shfl_xor_sync(0xffffffffu, c, 2);
              c += __shfl_xor_sync(0xffffffffu, c, 1);
              if ((lane & 3) == 0) {
                const int grp = (c0 >> 3) + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
                gacc[grp * 2 + (lane >> 4)] += c;
              }
            }
          }
          continue;
        }
        uint32_t raw[CH];
        acc_ld<CH>(acc_row + c0, raw);
        float v[CH];
#pragma unroll
        for (int j = 0; j < CH; ++j) v[j] = __uint_as_float(raw[j]);
        if (row_ok) epilogue_math<CH>(p, v, nb, ow, res_off, n0 + c0);
        if (p.stat_ptr && row_ok) {
          // online (max, sum exp) over this row's valid columns of the tile: softmax partials for the row pass
          float cmax = -INFINITY;
#pragma unroll
          for (int j = 0; j < CH; ++j)
            if (n0 + c0 + j < p.cout) cmax = fmaxf(cmax, v[j]);
          if (cmax > -INFINITY) {
            const float nm = fmaxf(run_max, cmax);
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < CH; ++j)
              if (n0 + c0 + j < p.cout) acc += __expf(v[j] - nm);
            run_sum = run_sum * __expf(run_max - nm) + acc;
            run_max = nm;
          }
        }
        if (p.out_staged) store_staged<CH>(p, v, my_tile, row_ok, out_off, n0 + c0, lane);
        else if (row_ok) store_direct<CH>(p, v, out_off, n0 + c0);
      }
      if (p.stat_ptr && row_ok) {
        float2* st = reinterpret_cast<float2*>(p.stat_ptr) + ((long long)ow * p.tiles_n + nt);
        *st = make_float2(run_max, run_sum);
      }
      if (want_key >= 0) {
#pragma unroll
        for (int i = 0; i < PER; ++i)
          if (lane + 32 * i < BN) addv_other[lane + 32 * i] = nbv[i] + nrw[i];
        next_key = want_key;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty_bar);
    }
    if (gn_on) { __syncwarp(); gn_flush(); }
  }

  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// The wide kernel: 128 x 256 tiles in clusters of two CTAs that share the weight tile
// ------------------------------------------------------------------------------------------------
// 384 threads: warpgroup 0 is the producer (one TMA thread; setmaxnreg hands its registers to the consumers), warpgroups
// 1 and 2 are consumers, each computing 64 rows x 256 columns with m64n256k16 (128 fp32 accumulators per thread) and
// running its own epilogue.  A work unit is a pair of adjacent M tiles with one 256-column tile; the two CTAs of a
// cluster take one M tile each.  Per 64-channel chunk a CTA loads its own 128 x 64 A box and one 128-row half of the
// 256 x 64 weight tile, multicast to both CTAs: against the 128-column kernel this halves the operand bytes per FLOP
// that leave L2 and the shared-memory bytes per FLOP that wgmma reads.  A ring slot's empty barrier takes one arrival
// per consumer warp of BOTH CTAs, because the peer's multicast writes into it.  While the consumers run the epilogue
// the producer already fills the ring with the next unit's chunks.
namespace wide {
static constexpr int kThreads = 384;
static constexpr int kCluster = 2;
static constexpr int kBN = 256;
static constexpr int kStages = 4;
static constexpr int kBHalfBytes = 128 * kBK * 2;                  // one CTA's share of the weight chunk: 16 KB
static constexpr int kStageBytes = kABytes + 2 * kBHalfBytes;      // 48 KB
static constexpr int kSliceLd = 36;                                // padded fp32 row of a 16 x 32 accumulator slice
static constexpr int kOffSlice = kStages * kStageBytes;            // per consumer warp: [16][kSliceLd] fp32
static constexpr int kOffAdd = kOffSlice + 8 * 16 * kSliceLd * 4;  // per consumer warp: bias + row vector [kBN] fp32
static constexpr int kOffBar = kOffAdd + 8 * kBN * 4;              // full[kStages], empty[kStages]
static constexpr int kSmem = 1024 + kOffBar + 2 * kStages * 8;
static constexpr int kProducerRegs = 40, kConsumerRegs = 232;
static_assert(kProducerRegs * 128 + kConsumerRegs * 256 <= 65536, "register budget of one CTA per SM");
}  // namespace wide

// GroupNorm partials of a 16-column chunk summed over the 16 lanes that share it (lane bits 0..3).  The lane then holds
// statistic (lane >> 3) & 1 (0 sum, 1 sum of squares) of group (lane >> 2) & 1 of the chunk (8-channel groups: gs[0..1]
// sums, gs[2..3] squares) or of group 2 ((lane >> 2) & 1) + ((lane >> 1) & 1) (4-channel groups: gs[0..3], gs[4..7]).
__device__ __forceinline__ float gn_reduce16(const float* gs, int lane, int gn_sh) {
  const bool h3 = (lane & 8) != 0, h2 = (lane & 4) != 0, h1 = (lane & 2) != 0;
  if (gn_sh == 3) {
    float a[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) a[i] = (h3 ? gs[2 + i] : gs[i]) + __shfl_xor_sync(0xffffffffu, h3 ? gs[i] : gs[2 + i], 8);
    float c = (h2 ? a[1] : a[0]) + __shfl_xor_sync(0xffffffffu, h2 ? a[0] : a[1], 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
  }
  float a4[4], a2[2];
#pragma unroll
  for (int i = 0; i < 4; ++i) a4[i] = (h3 ? gs[4 + i] : gs[i]) + __shfl_xor_sync(0xffffffffu, h3 ? gs[i] : gs[4 + i], 8);
#pragma unroll
  for (int i = 0; i < 2; ++i) a2[i] = (h2 ? a4[2 + i] : a4[i]) + __shfl_xor_sync(0xffffffffu, h2 ? a4[i] : a4[2 + i], 4);
  float c = (h1 ? a2[1] : a2[0]) + __shfl_xor_sync(0xffffffffu, h1 ? a2[0] : a2[1], 2);
  c += __shfl_xor_sync(0xffffffffu, c, 1);
  return c;
}

// Calls it takes (see wide_fits): h16 vector-aligned output with cout == out_cols a multiple of 256, h16 vector-aligned
// residual or none, no softmax statistics / GEGLU / row bias / batched weights / broadcast A / split-K.
// p.num_tiles is the number of units: ceil(M tiles / 2) x column tiles.
__global__ void __launch_bounds__(wide::kThreads, 1) igemm_wide_kernel(const __grid_constant__ IgemmDev p) {
  using namespace wide;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t ring = smem_u32(sm);
  const uint32_t full0 = ring + kOffBar, empty0 = full0 + 8 * kStages;

  const int tid = threadIdx.x;
  // warp-uniform by construction (broadcast from lane 0): otherwise ptxas treats the role branches as divergent and
  // serialises every wgmma behind them
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const uint32_t rank = cluster_ctarank();
  const int cid = (int)blockIdx.x / kCluster, n_clusters = (int)gridDim.x / kCluster;
  const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_d * p.N;
  const int num_units = p.num_tiles;
  const int num_k = p.num_k_chunks;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 8 * kCluster);     // one arrival per consumer warp of each CTA
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster_sync();                   // both CTAs' barriers exist before any multicast or remote arrival

  // unit u -> column tile u % tiles_n and M tile 2 (u / tiles_n) + rank (column tile fastest: neighbouring units share
  // their A halos in L2).  The partner of an odd last M tile loads a valid tile, runs the whole protocol, stores nothing.
  struct MTile { int nt, wt, ht, dt, nb; bool ok; };
  auto unit_tile = [&](int u) {
    MTile t;
    t.nt = u % p.tiles_n;
    int m = 2 * (u / p.tiles_n) + (int)rank;
    t.ok = m < m_tiles;
    if (!t.ok) m = m_tiles - 1;
    t.wt = m % p.tiles_w; m /= p.tiles_w;
    t.ht = m % p.tiles_h; m /= p.tiles_h;
    t.dt = m % p.tiles_d;
    t.nb = m / p.tiles_d;
    return t;
  };

  if (wg == 0) {
    // ============================== producer ==============================
    setmaxnreg_dec<kProducerRegs>();
    if (tid == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = cid; u < num_units; u += n_clusters) {
        const MTile t = unit_tile(u);
        const int iw0 = t.wt * p.BW * p.sw, ih0 = t.ht * p.BH * p.sh, id0 = t.dt * p.BD * p.sd;
        const int wrow = t.nt * kBN + 128 * (int)rank;      // this CTA's half of the weight tile
        int kglob = 0;
        for (int s = 0; s < p.n_seg; ++s) {
          const SegDev sg = p.seg[s];
          const CUtensorMap* tm = &p.tmA[sg.src];
          const int cw = iw0 + sg.dw, ch = ih0 + sg.dh, cd = id0 + sg.dd;
          for (int c = 0; c < sg.nchunks; ++c, ++kglob) {
            mbar_wait(empty0 + 8 * stage, phase ^ 1u);
            const uint32_t dst = ring + stage * kStageBytes, fb = full0 + 8 * stage;
            mbar_arrive_expect_tx(fb, kStageBytes);       // own A box + both halves of the weight chunk
            tma_load_5d(tm, fb, dst, (sg.c0 + c) * kBK, cw, ch, cd, t.nb);
            tma_load_3d_multicast(&p.tmB, fb, dst + kABytes + rank * kBHalfBytes, kglob * kBK, wrow, 0, 0x3);
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else {
    // ============================== consumers ==============================
    setmaxnreg_inc<kConsumerRegs>();
    const int c = wg - 1;                          // rows 64c .. 64c + 63 of the tile
    const int wq = (tid >> 5) & 3;                 // 16-row slice of those
    const int lane = tid & 31;
    float* slice = reinterpret_cast<float*>(sm + kOffSlice) + (4 * c + wq) * 16 * kSliceLd;
    float* addv = reinterpret_cast<float*>(sm + kOffAdd) + (4 * c + wq) * kBN;
    // epilogue: the lane owns row (lane & 15) of the warp's 16 rows and columns 16 (lane >> 4) .. + 15 of each
    // 32-column slice
    const int er = 64 * c + 16 * wq + (lane & 15);
    const int eh = lane >> 4;
    const int rw = er & (p.BW - 1), rh = (er >> p.bw_log2) & (p.BH - 1), rd = er >> (p.bw_log2 + p.bh_log2);
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive_cluster(empty0 + 8 * s, 0);
        mbar_arrive_cluster(empty0 + 8 * s, 1);
      }
    };

    // GroupNorm partials: gacc[s] is this lane's statistic (see gn_reduce16) of slice s, summed over the units of one
    // (sample, column tile); on a change it is added to slot gn_slot0 + 4 blockIdx.x + wq — the same slot for warp wq of
    // both consumers, so consumer 0 adds first and consumer 1 after a barrier (deterministic, no atomics)
    const bool gn_on = p.gn_partial != nullptr;
    const int gsh = p.gn_sh;
    float gacc[kBN / 32];
#pragma unroll
    for (int s = 0; s < kBN / 32; ++s) gacc[s] = 0.f;
    int key = -1, gn_nb = 0, gn_n0 = 0;
    auto gn_flush = [&]() {
      const bool writer = (lane & (gsh == 3 ? 3 : 1)) == 0;
      const int stat = (lane >> 3) & 1;
      const int gl = gsh == 3 ? (lane >> 2) & 1 : ((lane >> 1) & 3);
      float* dst = p.gn_partial +
                   (((long long)gn_nb * p.gn_slots + p.gn_slot0 + 4 * blockIdx.x + wq) * (p.cout >> gsh)) * 2 + stat;
      for (int pass = 0; pass < 2; ++pass) {
        if (pass == c && writer) {
#pragma unroll
          for (int s = 0; s < kBN / 32; ++s) dst[(((gn_n0 + 32 * s + 16 * eh) >> gsh) + gl) * 2] += gacc[s];
        }
        if (pass == 0) named_sync(1, 256);
      }
#pragma unroll
      for (int s = 0; s < kBN / 32; ++s) gacc[s] = 0.f;
    };

    float acc[kBN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int u = cid; u < num_units; u += n_clusters) {
      int prev = -1;
      for (int k = 0; k < num_k; ++k) {
        mbar_wait(full0 + 8 * stage, phase);
        const uint32_t st = ring + stage * kStageBytes;
        const uint64_t adesc = wgmma_desc(st + c * (64 * kBK * 2));
        const uint64_t bdesc = wgmma_desc(st + kABytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBK / 16; ++kk)
          wgmma_ss<kBN>(acc, adesc + 2u * kk, bdesc + 2u * kk, (k | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();            // the group of the previous chunk has finished reading its stage
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_touch<kBN / 2>(acc);
      release(prev);

      // ---- epilogue: the same arithmetic, in the same order, as the 128-column kernel's fast epilogue ----
      const MTile t = unit_tile(u);
      const int n0 = t.nt * kBN;
      const int ow = t.wt * p.BW + rw, oh = t.ht * p.BH + rh, od = t.dt * p.BD + rd;
      const bool row_ok = t.ok && ow < p.OW && oh < p.OH && od < p.OD;
      const long long out_off = t.nb * p.out_sN + od * p.out_sD + oh * p.out_sH + ow * p.out_sW;
      const long long res_off = t.nb * p.res_sN + od * p.res_sD + oh * p.res_sH + ow * p.res_sW;
      if (t.nb * p.tiles_n + t.nt != key) {
        if (gn_on && key >= 0) gn_flush();
        key = t.nb * p.tiles_n + t.nt;
        gn_nb = t.nb;
        gn_n0 = n0;
        // bias + per-sample row vector of this (sample, column tile), shared by all rows
        float bv[kBN / 32], rv[kBN / 32];
#pragma unroll
        for (int i = 0; i < kBN / 32; ++i) {
          const int col = n0 + lane + 32 * i;
          bv[i] = p.bias ? __ldg(p.bias + col) : 0.f;
          rv[i] = p.rowvec ? __ldg(p.rowvec + (long long)t.nb * p.rowvec_bstride + col) : 0.f;
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < kBN / 32; ++i) addv[lane + 32 * i] = bv[i] + rv[i];
        __syncwarp();
      }
      const bool res_on = p.res_ptr && row_ok;
      uint4 rv_next[2] = {make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u)};
      if (res_on) load_res_fast<16>(p, rv_next, res_off, n0 + 16 * eh);
#pragma unroll
      for (int s = 0; s < kBN / 32; ++s) {
        // the warp's 16 x 32 accumulator slice s through shared memory, so that a lane holds 16 columns of one row
        __syncwarp();
#pragma unroll
        for (int j = 4 * s; j < 4 * s + 4; ++j) {
          const int col = 8 * (j - 4 * s) + 2 * (lane & 3);
          *reinterpret_cast<float2*>(slice + (lane >> 2) * kSliceLd + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(slice + ((lane >> 2) + 8) * kSliceLd + col) =
              make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        __syncwarp();
        uint32_t raw[16];
        acc_ld<16>(slice + (lane & 15) * kSliceLd + 16 * eh, raw);
        const uint4 rv[2] = {rv_next[0], rv_next[1]};
        if (res_on && s + 1 < kBN / 32) load_res_fast<16>(p, rv_next, res_off, n0 + 32 * (s + 1) + 16 * eh);
        const int cc = 32 * s + 16 * eh;
        // (gs is always passed: a pointer select would keep it in local memory)
        float gs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (row_ok) epilogue_fast<16>(p, raw, addv + cc, rv, out_off, n0 + cc, gs);
        if (gn_on) gacc[s] += gn_reduce16(gs, lane, gsh);
      }
    }
    if (gn_on && key >= 0) gn_flush();
  }
  cluster_sync();                   // no CTA leaves while its partner may still multicast into it or arrive on its barriers
}

// ------------------------------------------------------------------------------------------------
// CUDA-core cross-check kernel: same parameters, same zero-fill semantics, same epilogue.
// One thread per (output voxel, 16-column group).  Used by tests and for debugging only.
// ------------------------------------------------------------------------------------------------
__global__ void igemm_check_kernel(const __grid_constant__ IgemmDev p) {
  const long long rows = (long long)p.N * p.OD * p.OH * p.OW;
  const int col_groups = (p.out_cols + 15) / 16;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * col_groups) return;
  const int cg = (int)(idx % col_groups);
  long long m = idx / col_groups;
  const int ow = (int)(m % p.OW); m /= p.OW;
  const int oh = (int)(m % p.OH); m /= p.OH;
  const int od = (int)(m % p.OD); m /= p.OD;
  const int nb = (int)m;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  const int wb = p.w_batched ? nb : 0;
  const h16* wbase = p.w_ptr + (long long)wb * p.w_bstride;
  int kglob = 0;
  for (int s = 0; s < p.n_seg; ++s) {
    const SegDev sg = p.seg[s];
    const int iw = ow * p.sw + sg.dw, ih = oh * p.sh + sg.dh, id = od * p.sd + sg.dd;
    const bool inb = iw >= 0 && iw < p.in_W && ih >= 0 && ih < p.in_H && id >= 0 && id < p.in_D;
    const h16* a = p.a_ptr[sg.src] +
        ((((long long)(p.a_bcast ? 0 : nb) * p.in_D + id) * p.in_H + ih) * p.in_W + iw) * p.a_pitch[sg.src];
    for (int c = 0; c < sg.nchunks; ++c, ++kglob) {
      if (!inb) continue;
      for (int e = 0; e < kBK; ++e) {
        const int ch = (sg.c0 + c) * kBK + e;
        const int kk = kglob * kBK + e;
        if (ch >= p.a_C[sg.src] || kk >= p.w_K) break;
        const float av = h2f(a[ch]);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = cg * 16 + j;
          if (col < p.w_rows) acc[j] += av * h2f(wbase[(long long)col * p.w_pitch + kk]);
        }
      }
    }
  }
  const long long out_off = nb * p.out_sN + od * p.out_sD + oh * p.out_sH + ow * p.out_sW;
  const long long res_off = nb * p.res_sN + od * p.res_sD + oh * p.res_sH + ow * p.res_sW;
  epilogue_row<16>(p, acc, nb, ow, out_off, res_off, cg * 16);
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled g_encode = nullptr;
static std::once_flag g_encode_once;

static void load_encode() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
      qres == cudaDriverEntryPointSuccess)
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
}

static int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

struct TileShape { int bw, bh, bd; };

// choose the 128-voxel box that wastes the fewest rows on this output extent
static TileShape choose_tile(int OW, int OH, int OD, int sw, int sh, int sd) {
  static const TileShape cands[] = {{128, 1, 1}, {64, 2, 1}, {32, 4, 1}, {16, 8, 1}, {8, 16, 1},
                                    {4, 32, 1},  {32, 2, 2}, {16, 4, 2}, {8, 8, 2},  {16, 2, 4},
                                    {8, 4, 4},   {4, 8, 4},  {4, 4, 8},  {8, 2, 8},  {2, 8, 8},
                                    {4, 2, 16},  {2, 4, 16}, {2, 2, 32}, {1, 1, 128}, {1, 128, 1},
                                    {2, 64, 1},  {1, 8, 16}, {1, 16, 8}};
  double best = 1e30;
  TileShape bt = cands[0];
  for (const TileShape& c : cands) {
    if (c.bw * sw > 256 || c.bh * sh > 256 || c.bd * sd > 256) continue;
    double tw = (double)((OW + c.bw - 1) / c.bw) * c.bw;
    double th = (double)((OH + c.bh - 1) / c.bh) * c.bh;
    double td = (double)((OD + c.bd - 1) / c.bd) * c.bd;
    double cost = tw * th * td;
    // prefer long contiguous runs along W on ties
    cost *= (1.0 + 1e-3 * (7 - ilog2(c.bw)));
    if (cost < best) { best = cost; bt = c; }
  }
  return bt;
}

// GroupNorm partials for the cross-check implementation: (sum, sumsq) of the stored bf16 outputs per 8-channel
// group, accumulated into slot gn_slot0 (fp32 atomics: test path only).
__global__ void gn8_partial_check_kernel(const __grid_constant__ IgemmDev p) {
  const long long rows = (long long)p.N * p.OD * p.OH * p.OW;
  const int gw = 1 << p.gn_sh;                      // channels per partial group (8 or 4)
  const int groups = p.cout >> p.gn_sh;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * groups) return;
  const int g = (int)(idx % groups);
  long long m = idx / groups;
  const int ow = (int)(m % p.OW); m /= p.OW;
  const int oh = (int)(m % p.OH); m /= p.OH;
  const int od = (int)(m % p.OD); m /= p.OD;
  const int nb = (int)m;
  const h16* o = reinterpret_cast<const h16*>(p.out_ptr) + nb * p.out_sN + od * p.out_sD +
                           oh * p.out_sH + ow * p.out_sW + g * gw;
  float s = 0.f, q = 0.f;
  for (int j = 0; j < gw; ++j) { const float f = h2f(o[j]); s += f; q = fmaf(f, f, q); }
  float* dst = p.gn_partial + (((long long)nb * p.gn_slots + p.gn_slot0) * groups + g) * 2;
  atomicAdd(dst, s);
  atomicAdd(dst + 1, q);
}

// Split-K second pass: one thread per (output row, 8-column group) sums the fp32 partials of the S reduction ranges
// in range order (deterministic) and applies the call's real epilogue — the same epilogue_math / store_direct the
// one-pass kernels use.
__global__ void __launch_bounds__(256) igemm_split_reduce_kernel(const IgemmDev p, const float* __restrict__ ws,
                                                                 int splits, int ws_cols, long long ws_stride) {
  const int groups = (p.out_cols + 7) >> 3;
  const long long rows = (long long)p.N * p.OD * p.OH * p.OW;
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= rows * groups) return;
  const int col0 = (int)(idx % groups) * 8;
  const long long row = idx / groups;
  long long t = row;
  const int ow = (int)(t % p.OW); t /= p.OW;
  const int oh = (int)(t % p.OH); t /= p.OH;
  const int od = (int)(t % p.OD); t /= p.OD;
  const int nb = (int)t;
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const float* src = ws + row * ws_cols + col0;
  int s = 0;
  // eight (then four) ranges' loads in flight per thread, additions in range order: the plain load -> add loop is one
  // L2 round trip per range
  for (; s + 8 <= splits; s += 8, src += 8 * ws_stride) {
    float4 a[8], b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      a[j] = __ldg(reinterpret_cast<const float4*>(src + j * ws_stride));
      b[j] = __ldg(reinterpret_cast<const float4*>(src + j * ws_stride + 4));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[0] += a[j].x; v[1] += a[j].y; v[2] += a[j].z; v[3] += a[j].w;
      v[4] += b[j].x; v[5] += b[j].y; v[6] += b[j].z; v[7] += b[j].w;
    }
  }
  if (s + 4 <= splits) {
    float4 a[4], b[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      a[j] = __ldg(reinterpret_cast<const float4*>(src + j * ws_stride));
      b[j] = __ldg(reinterpret_cast<const float4*>(src + j * ws_stride + 4));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[0] += a[j].x; v[1] += a[j].y; v[2] += a[j].z; v[3] += a[j].w;
      v[4] += b[j].x; v[5] += b[j].y; v[6] += b[j].z; v[7] += b[j].w;
    }
    s += 4; src += 4 * ws_stride;
  }
  if (s + 2 <= splits) {
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(src)), b0 = __ldg(reinterpret_cast<const float4*>(src + 4));
    const float4 a1 = __ldg(reinterpret_cast<const float4*>(src + ws_stride));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(src + ws_stride + 4));
    v[0] += a0.x; v[1] += a0.y; v[2] += a0.z; v[3] += a0.w; v[4] += b0.x; v[5] += b0.y; v[6] += b0.z; v[7] += b0.w;
    v[0] += a1.x; v[1] += a1.y; v[2] += a1.z; v[3] += a1.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
    s += 2; src += 2 * ws_stride;
  }
  if (s < splits) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(src));
    const float4 b = __ldg(reinterpret_cast<const float4*>(src + 4));
    v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w;
    v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
  }
  const long long out_off = nb * p.out_sN + od * p.out_sD + oh * p.out_sH + ow * p.out_sW;
  const long long res_off = nb * p.res_sN + od * p.res_sD + oh * p.res_sH + ow * p.res_sW;
  epilogue_math<8>(p, v, nb, ow, res_off, col0);
  store_direct<8>(p, v, out_off, col0);
}

// Launch geometry shared by b200_igemm and b200_igemm_split_workspace_bytes (host only, no CUDA calls but sm_count()).
struct Plan {
  TileShape ts;
  long long m_tiles, ntiles, rows;   // ntiles: work items of the launch (units of two M tiles for the wide kernel)
  int kchunks, BN, tiles_n;
  int splits, ws_cols;
  long long ws_bytes;
  bool wide;                         // igemm_wide_kernel (BN = 256)
};

// The calls igemm_wide_kernel can compute: its epilogue is the vectorised 16-bit one with every column real.
static bool wide_fits(const b200_igemm_params* p) {
  auto v8 = [](long long a, long long b, long long c, long long d) { return a % 8 == 0 && b % 8 == 0 && c % 8 == 0 && d % 8 == 0; };
  const bool out_vec = v8(p->out_sN, p->out_sD, p->out_sH, p->out_sW) && ((uintptr_t)p->out_ptr % 16) == 0;
  const bool res_ok = !p->res_ptr || (p->res_dtype == B200_DT_H16 && v8(p->res_sN, p->res_sD, p->res_sH, p->res_sW) &&
                                      ((uintptr_t)p->res_ptr % 16) == 0);
  return p->out_dtype == B200_DT_H16 && p->cout == p->out_cols && p->cout % wide::kBN == 0 && out_vec && res_ok &&
         !p->stat_ptr && p->act1 != B200_ACT_GEGLU && !p->row_bias && !p->w_batched && !p->a_broadcast;
}
// Reductions shorter than this many 64-channel chunks stay on the 128-column kernel, whose epilogue overlaps the next
// tile's main loop (the wide kernel's consumers run their own epilogue).
static constexpr int kWideMinChunks = 32;
// The shortest reduction, in 64-channel chunks, for which an under-filled grid narrows its column tile.
static constexpr int kNarrowMinChunks = 4;
// The fewest ranges a split reduction must have to be worth its fp32 partials and second kernel.
static constexpr int kSplitMin = 3;
// The shortest range, in chunks, a split may leave each CTA: a split only pays when every range still has ~2 000
// elements of reduction to hide its partial stores and the second kernel behind.
static constexpr int kSplitRangeMin = 32;
static Plan make_plan(const b200_igemm_params* p, bool allow_split, int nsm = 0) {
  if (nsm <= 0) nsm = sm_count();       // nsm > 0: the planning query of a machine of that size (no CUDA call at all)
  Plan pl;
  pl.kchunks = 0;
  for (int s = 0; s < p->n_seg; ++s) pl.kchunks += p->seg[s].nchunks;
  pl.ts = choose_tile(p->out_W, p->out_H, p->out_D, p->stride_w, p->stride_h, p->stride_d);
  const long long tw = (p->out_W + pl.ts.bw - 1) / pl.ts.bw, th = (p->out_H + pl.ts.bh - 1) / pl.ts.bh,
                  td = (p->out_D + pl.ts.bd - 1) / pl.ts.bd;
  pl.m_tiles = tw * th * td * p->out_N;
  pl.rows = (long long)p->out_N * p->out_D * p->out_H * p->out_W;
  pl.splits = 1;
  pl.ws_cols = ((p->out_cols + 7) / 8) * 8;
  pl.ws_bytes = 0;
  // 128 x 256 tiles in clusters of two (impl 3 forces them, impl 2 forbids them): convolutions (>= 8 taps) with a long
  // reduction whose units fill at least one wave of clusters.  GEMM-shaped calls keep the 128-column kernel.
  pl.wide = wide_fits(p) && (p->impl == 3 || (p->impl == 0 && p->n_seg >= 8 && pl.kchunks >= kWideMinChunks &&
                                            ((pl.m_tiles + 1) / 2) * (p->cout / wide::kBN) >= nsm / wide::kCluster));
  if (pl.wide) {
    pl.BN = wide::kBN;
    pl.tiles_n = p->cout / wide::kBN;
    pl.ntiles = ((pl.m_tiles + 1) / 2) * pl.tiles_n;
    return pl;
  }
  // N tile: as wide as the output needs, up to 128 columns (the widest tile whose fp32 hand-off buffer and a 4-deep
  // operand ring fit the 227 KB of shared memory a block may use)
  const int cols16 = (((p->act1 == B200_ACT_GEGLU ? p->cout : p->out_cols) + 15) / 16) * 16;   // GEGLU: tile the GEMM's columns
  int BN = cols16 <= 16 ? 16 : cols16 <= 32 ? 32 : cols16 <= 64 ? 64 : 128;
  if (p->stat_ptr) BN = 128;      // the caller sizes the partials buffer for 128-column tiles
  // A grid that cannot fill the SMs: keep the wide tile (operand traffic from L2 per FLOP falls with the tile width) and cut the
  // reduction into ranges instead, when the caller brought a workspace and the reduction is long enough for at least
  // two ranges of four 64-element chunks.
  const long long wide_tiles = pl.m_tiles * ((cols16 + BN - 1) / BN);
  if (allow_split && !p->stat_ptr && !p->gn_partial && p->impl != 1 && p->act1 != B200_ACT_GEGLU && pl.kchunks >= 16 &&
      wide_tiles * 2 <= nsm) {
    long long s = nsm / wide_tiles;
    if (s > pl.kchunks / kSplitRangeMin) s = pl.kchunks / kSplitRangeMin;
    if (s > 32) s = 32;
    if (s >= kSplitMin) {
      pl.splits = (int)s;
      pl.ws_bytes = s * pl.rows * pl.ws_cols * 4;
    }
  }
  // otherwise narrower tiles, down to 64 columns, to put more CTAs on the problem: halve the column tile while the
  // narrower tiles still fit ONE wave (a second wave of 64-column tiles streams every A tile four times from L2).  Short
  // reductions (K = 256 / 384: the transformer linears) are epilogue-bound and narrow the same way.
  if (pl.splits == 1) {
    while (!p->stat_ptr && BN > 64 && pl.kchunks >= kNarrowMinChunks &&
           pl.m_tiles * ((cols16 + BN / 2 - 1) / (BN / 2)) <= nsm) BN >>= 1;
  }
  pl.BN = BN;
  pl.tiles_n = (cols16 + BN - 1) / BN;
  pl.ntiles = pl.m_tiles * pl.tiles_n;
  return pl;
}

template <int BN, int STAGES>
static int launch_tc(const IgemmDev& d, cudaStream_t stream) {
  constexpr int kStageBytes = kABytes + BN * kBK * 2;
  constexpr int smem = 1024 + STAGES * kStageBytes + kBM * (BN + 4) * 4 + 256 + 4 * 32 * 33 * 4 + 8 * BN * 4;
  static_assert(smem <= 227 * 1024, "igemm: shared memory over the 227 KB a block may use");
  static std::once_flag attr_once;          // per instantiation; read-only afterwards (re-entrant entry point)
  static cudaError_t attr_rc = cudaSuccess;
  std::call_once(attr_once, [] {
    attr_rc = cudaFuncSetAttribute(igemm_tc_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  });
  B200_CUDA(attr_rc);
  const int grid = d.num_tiles < sm_count() ? d.num_tiles : sm_count();
  B200_CUDA(b200::launch_kernel(igemm_tc_kernel<BN, STAGES>, grid, kThreads, smem, stream, d));
  B200_LAUNCH_CHECK("igemm_tc_kernel");
  return B200_OK;
}

// persistent: at most as many clusters as can be co-resident, each walking units cid, cid + clusters, ...
static int launch_wide(const IgemmDev& d, cudaStream_t stream) {
  static_assert(wide::kSmem <= 227 * 1024, "igemm: shared memory over the 227 KB a block may use");
  static std::once_flag once;
  static cudaError_t rc = cudaSuccess;
  static int max_clusters = 0;
  std::call_once(once, [] {
    rc = cudaFuncSetAttribute(igemm_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, wide::kSmem);
    if (rc != cudaSuccess) return;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(wide::kCluster);
    cfg.blockDim = dim3(wide::kThreads);
    cfg.dynamicSmemBytes = wide::kSmem;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = wide::kCluster;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    rc = cudaOccupancyMaxActiveClusters(&max_clusters, igemm_wide_kernel, &cfg);
  });
  B200_CUDA(rc);
  if (max_clusters < 1) { set_error("igemm: no cluster of igemm_wide_kernel fits on this device"); return B200_ECUDA; }
  const int clusters = d.num_tiles < max_clusters ? d.num_tiles : max_clusters;
  B200_CUDA(b200::launch_kernel<wide::kCluster>(igemm_wide_kernel, clusters * wide::kCluster, wide::kThreads,
                                                wide::kSmem, stream, d));
  B200_LAUNCH_CHECK("igemm_wide_kernel");
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_igemm_split_workspace_bytes(const b200_igemm_params* p) {
  if (!p || p->n_seg < 1 || p->n_seg > B200_IGEMM_MAX_SEG || p->out_N < 1 || p->out_D < 1 || p->out_H < 1 ||
      p->out_W < 1 || p->out_cols < 1 || p->stride_d < 1 || p->stride_h < 1 || p->stride_w < 1)
    return 0;
  if (p->impl == 1) return 0;
  return make_plan(p, true).ws_bytes;
}

// Host-only planning query (no CUDA call): the column tile, the split factor and the tile count b200_igemm would use
// for this call on a GPU with `sm_count` SMs — lets the binding layer's CPU tests pin the planner's rules.  For calls
// of the wide kernel out[0] is 256 and out[2] the number of units (pairs of M tiles x column tiles).  out[3] is always 0.
extern "C" int b200_igemm_plan(const b200_igemm_params* p, int32_t sm_count_, int32_t with_workspace, int32_t out[4]) {
  if (!p || !out || sm_count_ < 1 || p->n_seg < 1 || p->n_seg > B200_IGEMM_MAX_SEG || p->out_N < 1 || p->out_D < 1 ||
      p->out_H < 1 || p->out_W < 1 || p->out_cols < 1)
    return B200_EINVAL;
  const Plan pl = make_plan(p, with_workspace != 0, sm_count_);
  out[0] = pl.BN;
  out[1] = pl.splits;
  out[2] = (int32_t)pl.ntiles;
  out[3] = 0;
  return B200_OK;
}

extern "C" int b200_igemm(const b200_igemm_params* p, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(p != nullptr, "igemm: null params");
  B200_CHECK_ARG(p->a_ptr[0] && p->w_ptr && p->out_ptr, "igemm: null tensor pointer");
  B200_CHECK_ARG(p->n_seg >= 1 && p->n_seg <= B200_IGEMM_MAX_SEG, "igemm: n_seg=%d out of range", p->n_seg);
  B200_CHECK_ARG(p->in_N >= 1 && p->in_D >= 1 && p->in_H >= 1 && p->in_W >= 1, "igemm: bad input extent");
  B200_CHECK_ARG(p->out_N == p->in_N && p->out_D >= 1 && p->out_H >= 1 && p->out_W >= 1, "igemm: bad output extent");
  const bool geglu = p->act1 == B200_ACT_GEGLU;
  B200_CHECK_ARG(p->cout >= 1 && p->out_cols >= (geglu ? p->cout / 2 : p->cout), "igemm: bad cout/out_cols");
  if (geglu) {
    B200_CHECK_ARG(p->cout % 64 == 0 && p->out_cols == p->cout / 2 && p->out_dtype == B200_DT_H16 && !p->res_ptr &&
                   p->scale == 1.0f && p->act2 == B200_ACT_NONE && !p->stat_ptr && !p->gn_partial && !p->row_bias &&
                   p->impl != 1,
                   "igemm: B200_ACT_GEGLU needs cout %% 64 == 0, out_cols == cout / 2, a h16 output and no residual / "
                   "scale / act2 / statistics / row bias (and has no cross-check kernel)");
  }
  B200_CHECK_ARG(p->w_pitch % 8 == 0 && p->w_rows >= 1, "igemm: weight pitch must be a multiple of 8");
  B200_CHECK_ARG(((uintptr_t)p->w_ptr & 15) == 0, "igemm: weight pointer not 16-byte aligned");
  B200_CHECK_ARG(p->stride_d >= 1 && p->stride_d <= 8 && p->stride_h >= 1 && p->stride_h <= 8 &&
                 p->stride_w >= 1 && p->stride_w <= 8, "igemm: stride out of range");
  for (int s = 0; s < 2; ++s) {
    if (!p->a_ptr[s]) continue;
    B200_CHECK_ARG(p->a_pitch[s] % 8 == 0 && p->a_C[s] >= 1 && p->a_C[s] <= p->a_pitch[s],
                   "igemm: source %d channel pitch %d / extent %d invalid", s, p->a_pitch[s], p->a_C[s]);
    B200_CHECK_ARG(((uintptr_t)p->a_ptr[s] & 15) == 0, "igemm: source %d not 16-byte aligned", s);
  }
  std::call_once(g_encode_once, load_encode);
  if (!g_encode) { set_error("igemm: cuTensorMapEncodeTiled entry point unavailable"); return B200_ECUDA; }

  IgemmDev d;
  memset(&d, 0, sizeof(d));
  int kchunks = 0;
  for (int s = 0; s < p->n_seg; ++s) {
    const b200_igemm_seg& sg = p->seg[s];
    B200_CHECK_ARG(sg.src == 0 || (sg.src == 1 && p->a_ptr[1]), "igemm: segment %d uses missing source", s);
    B200_CHECK_ARG(sg.nchunks >= 1, "igemm: segment %d has no chunks", s);
    d.seg[s].src = sg.src; d.seg[s].dw = sg.dw; d.seg[s].dh = sg.dh; d.seg[s].dd = sg.dd;
    d.seg[s].c0 = sg.c0; d.seg[s].nchunks = sg.nchunks;
    kchunks += sg.nchunks;
  }
  const int w_K = p->w_K > 0 ? p->w_K : p->w_pitch;   // K elements past w_K read as zero
  B200_CHECK_ARG(w_K <= p->w_pitch, "igemm: w_K %d exceeds the row pitch %d", w_K, p->w_pitch);
  d.n_seg = p->n_seg;
  d.num_k_chunks = kchunks;
  for (int s = 0; s < 2; ++s) {
    d.a_ptr[s] = reinterpret_cast<const h16*>(p->a_ptr[s]);
    d.a_C[s] = p->a_C[s];
    d.a_pitch[s] = p->a_pitch[s];
  }
  d.in_N = p->in_N; d.in_D = p->in_D; d.in_H = p->in_H; d.in_W = p->in_W;
  d.a_bcast = p->a_broadcast ? 1 : 0;
  d.w_ptr = reinterpret_cast<const h16*>(p->w_ptr);
  d.w_rows = p->w_rows; d.w_K = w_K; d.w_pitch = p->w_pitch;
  d.w_bstride = p->w_bstride; d.w_batched = p->w_batched;
  d.sd = p->stride_d; d.sh = p->stride_h; d.sw = p->stride_w;
  d.N = p->out_N; d.OD = p->out_D; d.OH = p->out_H; d.OW = p->out_W;
  d.out_ptr = p->out_ptr; d.out_dtype = p->out_dtype; d.cout = p->cout; d.out_cols = p->out_cols;
  d.out_sN = p->out_sN; d.out_sD = p->out_sD; d.out_sH = p->out_sH; d.out_sW = p->out_sW;
  d.bias = p->bias; d.rowvec = p->rowvec; d.rowvec_bstride = p->rowvec_bstride; d.row_bias = p->row_bias;
  d.act1 = geglu ? B200_ACT_NONE : p->act1; d.act2 = p->act2; d.scale = p->scale;
  d.geglu = geglu ? 1 : 0;
  if (geglu) d.out_cols = p->cout;        // the kernel's column loops run over the GEMM's columns
  d.res_ptr = p->res_ptr; d.res_dtype = p->res_dtype;
  d.res_sN = p->res_sN; d.res_sD = p->res_sD; d.res_sH = p->res_sH; d.res_sW = p->res_sW;
  {
    const int g = (p->out_dtype == B200_DT_H16) ? 8 : 4;
    d.out_vec = (p->out_cols % g == 0) && (p->out_sN % g == 0) && (p->out_sD % g == 0) &&
                (p->out_sH % g == 0) && (p->out_sW % g == 0) && (((uintptr_t)p->out_ptr) % 16 == 0);
    d.out_v256 = d.out_vec && p->out_dtype == B200_DT_H16 && (p->out_cols % 16 == 0) && (p->out_sN % 16 == 0) &&
                 (p->out_sD % 16 == 0) && (p->out_sH % 16 == 0) && (p->out_sW % 16 == 0) &&
                 (((uintptr_t)p->out_ptr) % 32 == 0);
  }
  B200_CHECK_ARG(!geglu || d.out_vec, "igemm: B200_ACT_GEGLU needs a 16-byte-aligned output (out_cols, strides %% 8 == 0)");
  {
    // rows far apart in memory (wide row-major GEMM outputs): stage the tile through smem for coalesced row stores
    const long long esz = (p->out_dtype == B200_DT_H16) ? 2 : 4;
    // (bf16 rows of 32 columns are already whole 64-byte segments per lane: those take the vectorised direct path)
    d.out_staged = (p->out_sW * esz > 2048 && p->out_dtype == B200_DT_F32) ? 1 : 0;
  }
  d.gn_partial = p->gn_partial; d.gn_slots = p->gn_slots; d.gn_slot0 = p->gn_slot0;
  B200_CHECK_ARG(p->gn_group == 0 || p->gn_group == 8 || p->gn_group == 4, "igemm: gn_group must be 8 (or 0) or 4");
  d.gn_sh = (p->gn_group == 4) ? 2 : 3;
  if (p->gn_partial) {
    // the partials ride on the vectorised epilogue: every column chunk must be a full 32-wide bf16 vector chunk
    B200_CHECK_ARG(p->out_dtype == B200_DT_H16 && p->cout % 32 == 0 && d.out_vec && !d.out_staged && !p->stat_ptr && p->gn_slot0 >= 0 && p->gn_slot0 + 4 * sm_count() <= p->gn_slots,
                   "igemm: gn_partial needs an h16 vector-aligned output with cout %% 32 == 0 and 4 x SM-count slots");
  }
  d.stat_ptr = p->stat_ptr;
  if (p->stat_ptr)
    B200_CHECK_ARG(p->out_N == 1 && p->out_D == 1 && p->out_H == 1, "igemm: stat_ptr needs a GEMM-shaped call");
  if (p->res_ptr) {
    const int g = (p->res_dtype == B200_DT_H16) ? 8 : 4;
    d.res_vec = (p->out_cols % g == 0) && (p->res_sN % g == 0) && (p->res_sD % g == 0) &&
                (p->res_sH % g == 0) && (p->res_sW % g == 0) && (((uintptr_t)p->res_ptr) % 16 == 0);
    d.res_v256 = d.res_vec && p->res_dtype == B200_DT_H16 && (p->out_cols % 16 == 0) && (p->res_sN % 16 == 0) &&
                 (p->res_sD % 16 == 0) && (p->res_sH % 16 == 0) && (p->res_sW % 16 == 0) &&
                 (((uintptr_t)p->res_ptr) % 32 == 0);
    B200_CHECK_ARG(!p->gn_partial || (d.res_vec && p->res_dtype == B200_DT_H16),
                   "igemm: gn_partial needs a vector-aligned h16 residual");
  }

  const int impl = p->impl;
  B200_CHECK_ARG(impl >= 0 && impl <= 3, "igemm: impl %d not in 0..3", impl);
  B200_CHECK_ARG(impl != 1 || !p->stat_ptr, "igemm: stat_ptr has no cross-check kernel (impl 1)");
  B200_CHECK_ARG(impl != 3 || wide_fits(p),
                 "igemm: impl 3 (128 x 256 tiles) needs a vector-aligned h16 output with cout == out_cols a multiple of "
                 "256, a vector-aligned h16 residual or none, and no stat_ptr / GEGLU / row_bias / batched weights / "
                 "broadcast A");
  if (impl == 1) {
    const long long rows = (long long)d.N * d.OD * d.OH * d.OW;
    const long long total = rows * ((d.out_cols + 15) / 16);
    const int threads = 128;
    const long long blocks = (total + threads - 1) / threads;
    B200_CHECK_ARG(blocks < (1ll << 31), "igemm(check): problem too large");
    B200_CUDA(b200::launch_kernel(igemm_check_kernel, (unsigned)blocks, threads, 0, stream, d));
    B200_LAUNCH_CHECK("igemm_check_kernel");
    if (d.gn_partial) {
      const long long tot = rows * (d.cout >> d.gn_sh);
      B200_CUDA(b200::launch_kernel(gn8_partial_check_kernel, (unsigned)((tot + 255) / 256), 256, 0, stream, d));
      B200_LAUNCH_CHECK("gn8_partial_check_kernel");
    }
    return B200_OK;
  }

  // ---- tile geometry ----
  const Plan pl = make_plan(p, p->split_ws != nullptr);
  const TileShape ts = pl.ts;
  d.BW = ts.bw; d.BH = ts.bh; d.BD = ts.bd;
  d.bw_log2 = ilog2(ts.bw); d.bh_log2 = ilog2(ts.bh);
  d.tiles_w = (d.OW + ts.bw - 1) / ts.bw;
  d.tiles_h = (d.OH + ts.bh - 1) / ts.bh;
  d.tiles_d = (d.OD + ts.bd - 1) / ts.bd;
  const int BN = pl.BN;
  d.tiles_n = pl.tiles_n;
  d.k_splits = 1;
  d.split_stride = 0;
  const int splits = (p->split_ws && pl.splits > 1) ? pl.splits : 1;
  if (splits > 1) {
    B200_CHECK_ARG(p->split_ws_bytes >= pl.ws_bytes && ((uintptr_t)p->split_ws & 15) == 0,
                   "igemm: split_ws needs %lld bytes, 16-byte aligned (got %lld)", pl.ws_bytes,
                   (long long)p->split_ws_bytes);
  }
  B200_CHECK_ARG(pl.ntiles * splits < (1ll << 31), "igemm: too many tiles");
  d.num_tiles = (int)pl.ntiles;

  // ---- tensor maps ----
  for (int s = 0; s < 2; ++s) {
    if (!p->a_ptr[s]) continue;
    cuuint64_t dims[5] = {(cuuint64_t)p->a_C[s], (cuuint64_t)p->in_W, (cuuint64_t)p->in_H,
                          (cuuint64_t)p->in_D, (cuuint64_t)(p->a_broadcast ? 1 : p->in_N)};
    const cuuint64_t pb = (cuuint64_t)p->a_pitch[s] * 2;
    cuuint64_t strides[4] = {pb, pb * p->in_W, pb * p->in_W * p->in_H,
                             pb * p->in_W * p->in_H * p->in_D};
    cuuint32_t box[5] = {(cuuint32_t)kBK, (cuuint32_t)(ts.bw * d.sw), (cuuint32_t)(ts.bh * d.sh),
                         (cuuint32_t)(ts.bd * d.sd), 1};
    cuuint32_t estr[5] = {1, (cuuint32_t)d.sw, (cuuint32_t)d.sh, (cuuint32_t)d.sd, 1};
    CUresult r = g_encode(&d.tmA[s], B200_H16_TMAP, 5, const_cast<void*>(p->a_ptr[s]),
                          dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("igemm: cuTensorMapEncodeTiled(A%d) failed with %d (C=%d pitch=%d in=%dx%dx%dx%d box=%ux%ux%u)",
                s, (int)r, p->a_C[s], p->a_pitch[s], p->in_N, p->in_D, p->in_H, p->in_W, box[1], box[2], box[3]);
      return B200_ECUDA;
    }
  }
  if (!p->a_ptr[1]) d.tmA[1] = d.tmA[0];
  {
    const int wbn = p->w_batched ? p->in_N : 1;
    cuuint64_t dims[3] = {(cuuint64_t)w_K, (cuuint64_t)p->w_rows, (cuuint64_t)wbn};
    cuuint64_t bs = p->w_bstride ? (cuuint64_t)p->w_bstride * 2 : (cuuint64_t)p->w_rows * p->w_pitch * 2;
    cuuint64_t strides[2] = {(cuuint64_t)p->w_pitch * 2, bs};
    B200_CHECK_ARG(bs % 16 == 0, "igemm: weight batch stride not 16-byte aligned");
    // the wide kernel loads its 256-row weight tile as two 128-row halves, one per CTA of the cluster
    cuuint32_t box[3] = {(cuuint32_t)kBK, (cuuint32_t)(pl.wide ? 128 : BN), 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = g_encode(&d.tmB, B200_H16_TMAP, 3, const_cast<void*>(p->w_ptr), dims,
                          strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("igemm: cuTensorMapEncodeTiled(W) failed with %d (K=%d rows=%d pitch=%d)", (int)r, w_K,
                p->w_rows, p->w_pitch);
      return B200_ECUDA;
    }
  }

  if (pl.wide) return launch_wide(d, stream);
  auto launch = [&](const IgemmDev& dev) {
    switch (BN) {
      case 16:  return launch_tc<16, 8>(dev, stream);
      case 32:  return launch_tc<32, 8>(dev, stream);
      case 64:  return launch_tc<64, 6>(dev, stream);
      default:  return launch_tc<128, 4>(dev, stream);
    }
  };
  if (splits == 1) return launch(d);

  // ---- split-K: S partial GEMMs into the fp32 workspace, then the reduction applies this call's epilogue ----
  IgemmDev ds = d;
  ds.k_splits = splits;
  ds.num_tiles = (int)(pl.ntiles * splits);
  ds.out_ptr = p->split_ws; ds.out_dtype = B200_DT_F32; ds.out_cols = pl.ws_cols;
  ds.out_sW = pl.ws_cols; ds.out_sH = ds.out_sW * d.OW; ds.out_sD = ds.out_sH * d.OH; ds.out_sN = ds.out_sD * d.OD;
  ds.split_stride = pl.rows * pl.ws_cols;
  ds.out_vec = 1; ds.out_v256 = 0;
  ds.out_staged = (ds.out_sW * 4 > 2048) ? 1 : 0;
  ds.bias = nullptr; ds.rowvec = nullptr; ds.row_bias = nullptr;
  ds.act1 = B200_ACT_NONE; ds.act2 = B200_ACT_NONE; ds.scale = 1.0f;
  ds.res_ptr = nullptr; ds.res_vec = 0; ds.res_v256 = 0;
  ds.stat_ptr = nullptr; ds.gn_partial = nullptr;
  const int rc = launch(ds);
  if (rc != B200_OK) return rc;
  const long long total = pl.rows * ((d.out_cols + 7) / 8);
  B200_CHECK_ARG((total + 255) / 256 < (1ll << 31), "igemm: split reduction too large");
  B200_CUDA(b200::launch_kernel(igemm_split_reduce_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, 
      d, static_cast<const float*>(p->split_ws), splits, pl.ws_cols, ds.split_stride));
  B200_LAUNCH_CHECK("igemm_split_reduce_kernel");
  return B200_OK;
}
