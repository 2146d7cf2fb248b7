// Flash-style attention on Hopper wgmma for every head_dim in {64, 128, 256, 512} (the large-T self-attention of the
// 3-D UNet: T = S = 89 600, one head of 512).
//
// Replaces torch.baddbmm -> softmax -> torch.bmm (diffusion_model_unet.py:143-153, 406-416; autoencoderkl.py:261-269),
// which materialise the T x S score matrix (29.9 GiB fp32 at T = 89 600).  Here the scores never leave the SM.
//
// head_dim <= 256, flash_attn_kernel<DCH>: one warpgroup per CTA, one CTA per (batch, head, 64-query tile)
//   per 64-key block:   S  = Q K^T        wgmma m64n64k16, A and B from shared memory, K = head_dim   -> registers
//                       P  = exp2(S*c - m) (fp32 online max / sum; a row lives in the four lanes of a quad)
//                       O += P V          wgmma m64nDk16, A = P straight from the S registers (16-bit), B = V^T tile
//   epilogue:           out = O / l (+ residual), 16-bit
// Q stays in shared memory for the whole tile; K and V^T have one buffer each: the next block's K is requested as soon
// as S has been computed (it lands during the softmax and PV), the next V^T as soon as PV has been issued and retired.
//
// head_dim 512, flash_attn_d512_kernel: a 64 x 512 fp32 accumulator does not fit one warpgroup's registers, so the CTA
// has two consumer warpgroups, each owning 256 of the output channels, and one producer warpgroup (one TMA thread;
// setmaxnreg moves its registers to the consumers).  Per 128-key block consumer c computes S for keys 64c .. 64c + 63
// only (S is computed once per block), the two exchange their row maxima and their 16-bit P tiles through shared
// memory, and each runs PV over all 128 keys for its own channels: A from registers for its own keys, from the
// partner's shared-memory P tile for the others.  K and V^T stream through a ring of 8 KB chunks (64 keys x 64
// channels) behind full / empty mbarriers; two CTAs on adjacent query tiles of one (batch, head) form a cluster and
// every chunk is multicast to both, so each chunk is read from L2 once per pair of query tiles.
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <mutex>
#include <string.h>

namespace b200 {

struct FlashDev {
  alignas(64) CUtensorMap tmQ;    // [B][T][C]      box (64 ch, 64 rows)
  alignas(64) CUtensorMap tmK;    // [B][S][C]      box (64 ch, 64 rows)
  alignas(64) CUtensorMap tmVt;   // [B][C][S]      box (64 keys, head_dim rows; 64 rows for head_dim 512)
  int B, T, S, heads, dh, d_chunks;
  int q_tiles, q_tiles_grid, n_items, n_kv;   // q_tiles_grid: CTAs per (batch, head), q_tiles rounded to the cluster
  float scale_log2;
  h16* out;
  long long out_bstride, out_pitch;
  const h16* res;
  long long res_bstride, res_pitch;
};

namespace fa {

static constexpr int kThreads = 128;
static constexpr int kBM = 64, kBKV = 64;
static constexpr int kChunkBytes = 64 * 64 * 2;        // 8 KB: 64 rows x 64 channels

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  h162 v = f2h2(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int DCH>      // DCH = head_dim / 64 (1, 2 or 4); the item computes all DV = head_dim output channels
__global__ void __launch_bounds__(kThreads, 1) flash_attn_kernel(const __grid_constant__ FlashDev p) {
  constexpr int DV = 64 * DCH;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t q_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t k_base = q_base + DCH * kChunkBytes;
  const uint32_t v_base = k_base + DCH * kChunkBytes;
  const uint32_t bar = v_base + DV * kBKV * 2;
  const uint32_t q_bar = bar, k_bar = bar + 8, v_bar = bar + 16;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  int x = blockIdx.x;
  const int qt = x % p.q_tiles; x /= p.q_tiles;
  const int h = x % p.heads;
  const int b = x / p.heads;
  const int q0 = qt * kBM;
  const int qc = h * p.dh;                  // first channel of this head
  const int vc = qc;                        // first output channel

  if (tid == 0) {
    mbar_init(q_bar, 1);
    mbar_init(k_bar, 1);
    mbar_init(v_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(q_bar, DCH * kChunkBytes);
    for (int c = 0; c < DCH; ++c) tma_load_3d(&p.tmQ, q_bar, q_base + c * kChunkBytes, qc + 64 * c, q0, b);
    mbar_arrive_expect_tx(k_bar, DCH * kChunkBytes);
    for (int c = 0; c < DCH; ++c) tma_load_3d(&p.tmK, k_bar, k_base + c * kChunkBytes, qc + 64 * c, 0, b);
    mbar_arrive_expect_tx(v_bar, DV * kBKV * 2);
    tma_load_3d(&p.tmVt, v_bar, v_base, 0, vc, b);
  }

  // rows r0 = 16 warp + lane / 4 and r0 + 8 of the tile; this lane's columns 8 j + 2 (lane % 4) + {0, 1}
  float o[DV / 2];
#pragma unroll
  for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // l: this lane's share of the row sums
  const float sc = p.scale_log2;
  mbar_wait(q_bar, 0);

  for (int j = 0; j < p.n_kv; ++j) {
    const uint32_t ph = j & 1;
    float s[32];
    mbar_wait(k_bar, ph);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < DCH; ++c) {
      const uint64_t qd = wgmma_desc(q_base + c * kChunkBytes), kd = wgmma_desc(k_base + c * kChunkBytes);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_ss<64>(s, qd + 2u * kk, kd + 2u * kk, (c | kk) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch<32>(s);
    __syncthreads();                          // every warp's S is done with the K buffer
    if (tid == 0 && j + 1 < p.n_kv) {
      mbar_arrive_expect_tx(k_bar, DCH * kChunkBytes);
      for (int c = 0; c < DCH; ++c) tma_load_3d(&p.tmK, k_bar, k_base + c * kChunkBytes, qc + 64 * c, (j + 1) * kBKV, b);
    }

    // online softmax in the log2 domain; keys past S (zero-filled by TMA) are masked out
    const int key0 = j * kBKV + 2 * (lane & 3);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = key0 + 8 * n + e < p.S;
        s[4 * n + e] = ok ? s[4 * n + e] * sc : -INFINITY;
        s[4 * n + 2 + e] = ok ? s[4 * n + 2 + e] * sc : -INFINITY;
        mx0 = fmaxf(mx0, s[4 * n + e]);
        mx1 = fmaxf(mx1, s[4 * n + 2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float nm0 = fmaxf(m0, mx0), nm1 = fmaxf(m1, mx1);
    // a row with no valid key so far keeps a finite reference so that no inf - inf appears
    const float u0 = nm0 == -INFINITY ? 0.f : nm0, u1 = nm1 == -INFINITY ? 0.f : nm1;
    const float a0 = ex2_approx(m0 - u0), a1 = ex2_approx(m1 - u1);
    m0 = nm0;
    m1 = nm1;
    uint32_t pa[16];
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const float p00 = ex2_approx(s[4 * n] - u0), p01 = ex2_approx(s[4 * n + 1] - u0);
      const float p10 = ex2_approx(s[4 * n + 2] - u1), p11 = ex2_approx(s[4 * n + 3] - u1);
      ps0 += p00 + p01;
      ps1 += p10 + p11;
      // A fragment of k16 step n / 2: {row r0, k lo}, {row r0 + 8, k lo}, {row r0, k hi}, {row r0 + 8, k hi}
      pa[4 * (n >> 1) + 2 * (n & 1)] = pack_h2(p00, p01);
      pa[4 * (n >> 1) + 2 * (n & 1) + 1] = pack_h2(p10, p11);
    }
    l0 = l0 * a0 + ps0;
    l1 = l1 * a1 + ps1;
#pragma unroll
    for (int n = 0; n < DV / 8; ++n) {
      o[4 * n] *= a0; o[4 * n + 1] *= a0;
      o[4 * n + 2] *= a1; o[4 * n + 3] *= a1;
    }

    mbar_wait(v_bar, ph);
    wgmma_fence();
    const uint64_t vd = wgmma_desc(v_base);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs<DV>(o, pa + 4 * kk, vd + 2u * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch<DV / 2>(o);
    __syncthreads();                          // every warp's PV is done with the V^T buffer
    if (tid == 0 && j + 1 < p.n_kv) {
      mbar_arrive_expect_tx(v_bar, DV * kBKV * 2);
      tma_load_3d(&p.tmVt, v_bar, v_base, (j + 1) * kBKV, vc, b);
    }
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  const int r0 = 16 * warp + (lane >> 2);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int t = q0 + r0 + 8 * half;
    if (t >= p.T) continue;
    const float inv = half ? inv1 : inv0;
    h16* orow = p.out + (long long)b * p.out_bstride + (long long)t * p.out_pitch + vc;
    const h16* rrow = p.res ? p.res + (long long)b * p.res_bstride + (long long)t * p.res_pitch + vc : nullptr;
#pragma unroll
    for (int n = 0; n < DV / 8; ++n) {
      const int col = 8 * n + 2 * (lane & 3);
      float v0 = o[4 * n + 2 * half] * inv, v1 = o[4 * n + 2 * half + 1] * inv;
      if (rrow) {
        const float2 r = h22f2(*reinterpret_cast<const h162*>(rrow + col));
        v0 += r.x;
        v1 += r.y;
      }
      *reinterpret_cast<h162*>(orow + col) = f2h2(v0, v1);
    }
  }
}

template <int DCH>
constexpr int smem_bytes() { return 1024 + 2 * DCH * kChunkBytes + DCH * 64 * kBKV * 2 + 64; }

// ------------------------------------------------------------------------------------------------ head_dim 512
namespace d512 {
static constexpr int kThreads = 384;              // warpgroup 0: producer; warpgroups 1, 2: consumers 0, 1
static constexpr int kCluster = 2;                // CTAs on adjacent query tiles sharing every K / V^T chunk
static constexpr int kBlockKeys = 128;                  // keys per block, 64 per consumer
static constexpr int kRing = 16;                  // ring slots of one 8 KB chunk; a key block streams 32 chunks
static constexpr int kChunksPerBlock = 32;
static constexpr int kOffRing = 8 * kChunkBytes;                   // Q: 8 chunks of 64 rows x 64 channels
static constexpr int kOffP = kOffRing + kRing * kChunkBytes;       // P tiles of consumers 0, 1: 64 rows x 64 keys
static constexpr int kOffX = kOffP + 2 * kChunkBytes;              // float row maxima [2][64], row sums [2][64]
static constexpr int kOffBar = kOffX + 4 * 64 * 4;                 // Q barrier, full[kRing], empty[kRing]
static constexpr int kSmem = 1024 + kOffBar + (1 + 2 * kRing) * 8;
static constexpr int kProducerRegs = 40, kConsumerRegs = 232;      // 128 x 40 + 256 x 232 <= 64 K registers
static_assert(kProducerRegs * 128 + kConsumerRegs * 256 <= 65536, "register budget of one CTA per SM");
}  // namespace d512

// Chunk n (0..31) of key block j, in ring slot n % 16 (each slot is used by one K and one V^T chunk per block):
//   n < 16:  K,   consumer c = (n / 4) % 2, keys j*128 + 64 c .. +63, channels 64 d .. +63 with
//                 depth chunk d = n % 4 + 4 (n / 8)
//   n >= 16: V^T, group g = (n - 16) / 4: keys j*128 + 64 (g / 2) .. +63,
//                 channels 256 (g % 2) + 64 ((n - 16) % 4) .. +63                       -> consumer g % 2
// So slots 4c .. 4c + 3 and 8 + 4c .. 11 + 4c only ever hold chunks of consumer c, which waits for every phase of
// its slots in order (a barrier can never be a whole phase ahead of its only reader).  A V^T group's four chunks are
// four consecutive 1024-byte-aligned slots, i.e. one 256-row B operand of m64n256k16.  Chunk n is loaded by CTA n % 2
// of the cluster and multicast to both; every CTA's producer arms its own full barrier for every chunk, and a slot's
// empty barrier takes one arrival per consuming warp in each of the two CTAs.
__global__ void __launch_bounds__(d512::kThreads, 1) flash_attn_d512_kernel(const __grid_constant__ FlashDev p) {
  using namespace d512;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t base = smem_u32(sm);
  const uint32_t q_base = base, ring = base + kOffRing, p_base = base + kOffP;
  float* xmax = reinterpret_cast<float*>(sm + kOffX);          // [consumer][row]
  float* xsum = xmax + 2 * 64;
  const uint32_t q_bar = base + kOffBar;
  const uint32_t full0 = q_bar + 8, empty0 = full0 + 8 * kRing;

  const int tid = threadIdx.x;
  // warp-uniform by construction (broadcast from lane 0): otherwise ptxas treats the role branches as divergent and
  // serialises every wgmma behind them
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const uint32_t rank = cluster_ctarank();
  int x = blockIdx.x;
  const int qt = x % p.q_tiles_grid; x /= p.q_tiles_grid;
  const int h = x % p.heads;
  const int b = x / p.heads;
  // the partner of an odd last tile has no rows: it loads a valid tile and runs the whole protocol but stores nothing
  const bool rows_valid = qt < p.q_tiles;
  const int q0 = (rows_valid ? qt : p.q_tiles - 1) * kBM;
  const int qc = h * 512;

  if (tid == 0) {
    mbar_init(q_bar, 1);
    for (int s = 0; s < kRing; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 4 * kCluster);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster_sync();                             // both CTAs' barriers exist before any multicast or remote arrival

  if (wg == 0) {
    // ---------------------------------------------------------------- producer
    setmaxnreg_dec<kProducerRegs>();
    if (tid == 0) {
      mbar_arrive_expect_tx(q_bar, 8 * kChunkBytes);
      for (int c = 0; c < 8; ++c) tma_load_3d(&p.tmQ, q_bar, q_base + c * kChunkBytes, qc + 64 * c, q0, b);
      for (int j = 0; j < p.n_kv; ++j) {
        for (int n = 0; n < kChunksPerBlock; ++n) {
          const int slot = n % kRing;
          // use 2j + n / 16 of the slot waits for the release of use 2j + n / 16 - 1 (the first wait passes)
          mbar_wait(empty0 + 8 * slot, ((n / kRing) & 1) ^ 1);
          mbar_arrive_expect_tx(full0 + 8 * slot, kChunkBytes);
          if ((n & 1) != (int)rank) continue;
          const uint32_t dst = ring + slot * kChunkBytes, fb = full0 + 8 * slot;
          if (n < 16) {
            const int d = (n & 3) | ((n >> 3) << 2);
            tma_load_3d_multicast(&p.tmK, fb, dst, qc + 64 * d, j * kBlockKeys + 64 * ((n >> 2) & 1), b, 0x3);
          } else {
            const int g = (n - 16) >> 2;
            tma_load_3d_multicast(&p.tmVt, fb, dst, j * kBlockKeys + 64 * (g >> 1), qc + 256 * (g & 1) + 64 * (n & 3), b,
                                  0x3);
          }
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumer c
    setmaxnreg_inc<kConsumerRegs>();
    const int c = wg - 1;
    const int t = tid & 127, warp = t >> 5, lane = tid & 31, q4 = lane & 3;
    const int r0 = 16 * warp + (lane >> 2);                    // this lane's rows r0 and r0 + 8
    const int sw = r0 & 7;                                     // 128-byte swizzle phase of both rows
    uint32_t* pmine = reinterpret_cast<uint32_t*>(sm + kOffP + c * kChunkBytes);
    const uint64_t pd_partner = wgmma_desc(p_base + (1 - c) * kChunkBytes);
    auto release = [&](int slot) {
      if (lane == 0) {
        mbar_arrive_cluster(empty0 + 8 * slot, 0);
        mbar_arrive_cluster(empty0 + 8 * slot, 1);
      }
    };

    float o[128];                                              // 64 rows x 256 channels 256c .. 256c + 255
#pragma unroll
    for (int i = 0; i < 128; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // l: this lane's share of the sums over own keys
    const float sc = p.scale_log2;
    mbar_wait(q_bar, 0);

    for (int j = 0; j < p.n_kv; ++j) {
      // S = Q K_c^T over the 8 depth chunks; a chunk is released once the group that read it has retired
      float s[32];
      auto k_slot = [c](int d) { return (d & 3) | (c << 2) | ((d >> 2) << 3); };
#pragma unroll
      for (int d = 0; d < 8; ++d) {
        const int slot = k_slot(d);
        mbar_wait(full0 + 8 * slot, 0);
        if (d == 0) wgmma_fence();
        const uint64_t qd = wgmma_desc(q_base + d * kChunkBytes), kd = wgmma_desc(ring + slot * kChunkBytes);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss<64>(s, qd + 2u * kk, kd + 2u * kk, (d | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        if (d >= 2) {
          wgmma_wait<2>();
          release(k_slot(d - 2));
        }
      }
      wgmma_wait<1>();
      release(k_slot(6));
      wgmma_wait<0>();
      release(k_slot(7));
      wgmma_touch<32>(s);

      // online softmax in the log2 domain over both halves of the block; keys past S are masked out
      const int key0 = j * kBlockKeys + 64 * c + 2 * q4;
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool ok = key0 + 8 * n + e < p.S;
          s[4 * n + e] = ok ? s[4 * n + e] * sc : -INFINITY;
          s[4 * n + 2 + e] = ok ? s[4 * n + 2 + e] * sc : -INFINITY;
          mx0 = fmaxf(mx0, s[4 * n + e]);
          mx1 = fmaxf(mx1, s[4 * n + 2 + e]);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      if (q4 == 0) {
        xmax[64 * c + r0] = mx0;
        xmax[64 * c + r0 + 8] = mx1;
      }
      named_sync(1, 256);                     // both consumers' block maxima are posted
      mx0 = fmaxf(mx0, xmax[64 * (1 - c) + r0]);
      mx1 = fmaxf(mx1, xmax[64 * (1 - c) + r0 + 8]);
      const float nm0 = fmaxf(m0, mx0), nm1 = fmaxf(m1, mx1);
      // a row with no valid key so far keeps a finite reference so that no inf - inf appears
      const float u0 = nm0 == -INFINITY ? 0.f : nm0, u1 = nm1 == -INFINITY ? 0.f : nm1;
      const float a0 = ex2_approx(m0 - u0), a1 = ex2_approx(m1 - u1);
      m0 = nm0;
      m1 = nm1;
      uint32_t pa[16];
      float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const float p00 = ex2_approx(s[4 * n] - u0), p01 = ex2_approx(s[4 * n + 1] - u0);
        const float p10 = ex2_approx(s[4 * n + 2] - u1), p11 = ex2_approx(s[4 * n + 3] - u1);
        ps0 += p00 + p01;
        ps1 += p10 + p11;
        // A fragment of k16 step n / 2: {row r0, k lo}, {row r0 + 8, k lo}, {row r0, k hi}, {row r0 + 8, k hi}
        const uint32_t lo = pack_h2(p00, p01), hi = pack_h2(p10, p11);
        pa[4 * (n >> 1) + 2 * (n & 1)] = lo;
        pa[4 * (n >> 1) + 2 * (n & 1) + 1] = hi;
        // the same values as the partner's A operand: K-major 128-byte-swizzled 64 x 64 tile
        pmine[(r0 * 128 + ((n ^ sw) << 4) + 4 * q4) >> 2] = lo;
        pmine[((r0 + 8) * 128 + ((n ^ sw) << 4) + 4 * q4) >> 2] = hi;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the P tile is read by the partner's wgmma
      l0 = l0 * a0 + ps0;
      l1 = l1 * a1 + ps1;
#pragma unroll
      for (int n = 0; n < 32; ++n) {
        o[4 * n] *= a0; o[4 * n + 1] *= a0;
        o[4 * n + 2] *= a1; o[4 * n + 3] *= a1;
      }
      named_sync(1, 256);                     // both P tiles are written

      // O += P V over keys half 0, then half 1: own half with A from registers, the partner's from its P tile
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int g = 2 * hh + c;             // V^T group: keys half hh, channels of consumer c, slots 4g .. 4g + 3
#pragma unroll
        for (int i = 0; i < 4; ++i) mbar_wait(full0 + 8 * (4 * g + i), 1);
        if (hh == 0) wgmma_fence();
        const uint64_t vd = wgmma_desc(ring + 4 * g * kChunkBytes);
        if (hh == c) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_rs<256>(o, pa + 4 * kk, vd + 2u * kk, 1u);
        } else {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_ss<256>(o, pd_partner + 2u * kk, vd + 2u * kk, 1u);
        }
        wgmma_commit();
      }
      wgmma_wait<1>();
#pragma unroll
      for (int i = 0; i < 4; ++i) release(4 * c + i);
      wgmma_wait<0>();
      wgmma_touch<128>(o);
      wgmma_touch_u32<16>(pa);
#pragma unroll
      for (int i = 0; i < 4; ++i) release(4 * (2 + c) + i);
    }

    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    if (q4 == 0) {
      xsum[64 * c + r0] = l0;
      xsum[64 * c + r0 + 8] = l1;
    }
    named_sync(1, 256);
    const float inv0 = 1.f / (l0 + xsum[64 * (1 - c) + r0]), inv1 = 1.f / (l1 + xsum[64 * (1 - c) + r0 + 8]);
    const int vc = qc + 256 * c;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int tq = q0 + r0 + 8 * half;
      if (!rows_valid || tq >= p.T) continue;
      const float inv = half ? inv1 : inv0;
      h16* orow = p.out + (long long)b * p.out_bstride + (long long)tq * p.out_pitch + vc;
      const h16* rrow = p.res ? p.res + (long long)b * p.res_bstride + (long long)tq * p.res_pitch + vc : nullptr;
#pragma unroll
      for (int n = 0; n < 32; ++n) {
        const int col = 8 * n + 2 * q4;
        float v0 = o[4 * n + 2 * half] * inv, v1 = o[4 * n + 2 * half + 1] * inv;
        if (rrow) {
          const float2 r = h22f2(*reinterpret_cast<const h162*>(rrow + col));
          v0 += r.x;
          v1 += r.y;
        }
        *reinterpret_cast<h162*>(orow + col) = f2h2(v0, v1);
      }
    }
  }
  cluster_sync();                             // no CTA leaves while its partner may still arrive on its barriers
}

static PFN_cuTensorMapEncodeTiled g_encode = nullptr;
static std::once_flag g_once;
static void load_encode() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
      qres == cudaDriverEntryPointSuccess)
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
}

static int encode3(CUtensorMap* tm, const void* ptr, cuuint64_t d0, cuuint64_t d1, cuuint64_t d2, cuuint64_t s1_bytes,
                   cuuint64_t s2_bytes, cuuint32_t b0, cuuint32_t b1, const char* what) {
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1_bytes, s2_bytes};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(tm, B200_H16_TMAP, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("attention_flash: cuTensorMapEncodeTiled(%s) failed with %d", what, (int)r);
    return B200_ECUDA;
  }
  return B200_OK;
}

template <int DCH>
static int launch(const FlashDev& d, cudaStream_t stream) {
  constexpr int smem = smem_bytes<DCH>();
  static_assert(smem <= 227 * 1024, "attention_flash: shared memory over the 227 KB a block may use");
  static std::once_flag attr_once;
  static cudaError_t attr_rc = cudaSuccess;
  std::call_once(attr_once, [] {
    attr_rc = cudaFuncSetAttribute(flash_attn_kernel<DCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  });
  B200_CUDA(attr_rc);
  B200_CUDA(b200::launch_kernel(flash_attn_kernel<DCH>, d.n_items, kThreads, smem, stream, d));
  B200_LAUNCH_CHECK("flash_attn_kernel");
  return B200_OK;
}

static int launch_d512(const FlashDev& d, cudaStream_t stream) {
  static_assert(d512::kSmem <= 227 * 1024, "attention_flash: shared memory over the 227 KB a block may use");
  static std::once_flag attr_once;
  static cudaError_t attr_rc = cudaSuccess;
  std::call_once(attr_once, [] {
    attr_rc = cudaFuncSetAttribute(flash_attn_d512_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, d512::kSmem);
  });
  B200_CUDA(attr_rc);
  B200_CUDA(b200::launch_kernel<d512::kCluster>(flash_attn_d512_kernel, d.n_items, d512::kThreads, d512::kSmem, stream, d));
  B200_LAUNCH_CHECK("flash_attn_d512_kernel");
  return B200_OK;
}

}  // namespace fa
}  // namespace b200

using namespace b200;

// No workspace: the kernels keep every probability tile on chip.
extern "C" int64_t b200_attention_flash_workspace_bytes(const b200_flash_params* a) {
  (void)a;
  return 0;
}

extern "C" int b200_attention_flash(const b200_flash_params* a, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  B200_CHECK_ARG(a && a->q && a->k && a->vt && a->out, "attention_flash: null pointer");
  B200_CHECK_ARG(a->B >= 1 && a->T >= 1 && a->S >= 1 && a->heads >= 1, "attention_flash: bad extents");
  B200_CHECK_ARG(a->dh == 64 || a->dh == 128 || a->dh == 256 || a->dh == 512,
                 "attention_flash: head_dim %d not in {64,128,256,512}", a->dh);
  B200_CHECK_ARG(a->q_pitch % 8 == 0 && a->k_pitch % 8 == 0 && a->vt_pitch % 8 == 0 && a->out_pitch % 8 == 0,
                 "attention_flash: pitches must be multiples of 8 elements");
  B200_CHECK_ARG(((uintptr_t)a->q & 15) == 0 && ((uintptr_t)a->k & 15) == 0 && ((uintptr_t)a->vt & 15) == 0 &&
                 ((uintptr_t)a->out & 15) == 0 && ((uintptr_t)a->res & 15) == 0, "attention_flash: 16-byte alignment");
  B200_CHECK_ARG(!a->res || a->res_pitch % 8 == 0, "attention_flash: residual pitch must be a multiple of 8");
  std::call_once(fa::g_once, fa::load_encode);
  if (!fa::g_encode) { set_error("attention_flash: cuTensorMapEncodeTiled unavailable"); return B200_ECUDA; }

  FlashDev d;
  memset(&d, 0, sizeof(d));
  const int C = a->heads * a->dh;
  const bool d512 = a->dh == 512;
  d.B = a->B; d.T = a->T; d.S = a->S; d.heads = a->heads; d.dh = a->dh;
  d.d_chunks = a->dh / 64;
  d.q_tiles = (a->T + fa::kBM - 1) / fa::kBM;
  d.q_tiles_grid = d512 ? (d.q_tiles + fa::d512::kCluster - 1) / fa::d512::kCluster * fa::d512::kCluster : d.q_tiles;
  const int bkv = d512 ? fa::d512::kBlockKeys : fa::kBKV;
  d.n_kv = (a->S + bkv - 1) / bkv;
  const long long items = (long long)a->B * a->heads * d.q_tiles_grid;
  B200_CHECK_ARG(items < (1ll << 31), "attention_flash: too many work items");
  d.n_items = (int)items;
  d.scale_log2 = a->scale * 1.4426950408889634f;
  d.out = reinterpret_cast<h16*>(a->out);
  d.out_pitch = a->out_pitch; d.out_bstride = (long long)a->T * a->out_pitch;
  d.res = reinterpret_cast<const h16*>(a->res);
  d.res_pitch = a->res_pitch; d.res_bstride = (long long)a->T * a->res_pitch;
  int rc;
  if ((rc = fa::encode3(&d.tmQ, a->q, C, a->T, a->B, (cuuint64_t)a->q_pitch * 2, (cuuint64_t)a->T * a->q_pitch * 2, 64,
                        fa::kBM, "Q"))) return rc;
  if ((rc = fa::encode3(&d.tmK, a->k, C, a->S, a->B, (cuuint64_t)a->k_pitch * 2, (cuuint64_t)a->S * a->k_pitch * 2, 64,
                        fa::kBKV, "K"))) return rc;
  if ((rc = fa::encode3(&d.tmVt, a->vt, a->S, C, a->B, (cuuint64_t)a->vt_pitch * 2, (cuuint64_t)C * a->vt_pitch * 2,
                        fa::kBKV, d512 ? 64 : a->dh, "V^T"))) return rc;
  switch (d.d_chunks) {
    case 1: return fa::launch<1>(d, stream);
    case 2: return fa::launch<2>(d, stream);
    case 4: return fa::launch<4>(d, stream);
    default: return fa::launch_d512(d, stream);
  }
}
