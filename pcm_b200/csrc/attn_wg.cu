// Flash attention on Hopper warpgroup MMA (sm_90a).  Forward for head sizes d <= 128 (SD1.5 / SDXL: 40,
// 64, 80).  One CTA = 128 query rows of one (batch, head): warpgroup 0 is the TMA producer (one
// thread), warpgroups 1 and 2 each own 64 query rows.  Q is loaded once; 64-key K / V tiles stream
// through a two-stage mbarrier ring.  S = Q K^T (wgmma, both operands K-major from shared memory)
// and O (m64 x 64 per 64-column block) live in the consumers' registers; P = exp2(c S - m) is packed
// to bf16 in registers and fed to O += P V as the register A operand, V read MN-major from the tile
// TMA wrote.  Head columns are handled in 64-wide blocks (KB = 1 for d <= 64, 2 for d <= 128); the
// columns of a block past d belong to the next head (or lie outside the tensor map and read as zero):
// they are zeroed in Q, so they add nothing to S, and the matching O columns are not stored.
// Keys past Skv (zero rows of the tensor map) are masked to -inf in the last block of a ragged Skv.
//
// Same contract as attn_fwd_kernel (attn.cu): q [B, Sq, H*D] (row stride ldq), k / v [B, Skv, H*D],
// out like q, lse [B, H, Sq] in log2 units of the scaled scores.
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"
#include "host_common.h"

namespace pcm {

namespace {

constexpr int kAwThreads = 384;
constexpr int kAwStages = 2;    // K / V ring of the forward
constexpr int kBwdStages = 3;   // streamed Q / dO or K / V ring of the backward
constexpr int kTile = 64 * 128;  // 64 rows x 64 bf16, SWIZZLE_128B

struct alignas(64) AttnWgParams {
  CUtensorMap q_map, k_map, v_map;
  bf16* out;
  float* lse;
  int H, Sq, Skv, D;
  long long ldo;
  float c;  // scale * log2(e)
};

// Keep a register A operand of an in-flight wgmma live and unchanged until its group has been waited for.
__device__ __forceinline__ void keep_operand(uint32_t (&a)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) asm volatile("" : "+r"(a[i][k])::"memory");
}

// P (fp32, in the accumulator fragment) -> bf16 register A operands of 4 k-steps of 16 keys
__device__ __forceinline__ void pack_operand(uint32_t (&a)[4][4], const float (&x)[32]) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) a[i >> 3][(i & 7) >> 1] = pack_bf16x2(x[i], x[i + 1]);
}

// Online softmax of one 64-key block on the S accumulator fragment (rows r and r + 8 of the thread; a
// row lives in one quad of lanes).  s becomes c S, with keys from kbase on past Skv at -inf when MASK;
// m_run takes the block's row maxima, alpha the factors that rescale the old row state, rs the block's
// row sums of P = exp2(c S - m), and pa P as register A operands of 4 k-steps of 16 keys.
// The scale and the subtraction round separately (no FFMA), as they did when the mask's select stood
// between them; exp2_ftz only drops P / alpha below 2^-126, weights that cannot move a row sum whose
// largest term is 1.
template <bool MASK>
__device__ __forceinline__ void fwd_softmax(float (&s)[32], float (&m_run)[2], float (&alpha)[2], float (&rs)[2],
                                            uint32_t (&pa)[4][4], float c, int kbase, int Skv) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    float v = __fmul_rn(s[i], c);
    if (MASK && kbase + 8 * (i >> 2) + (i & 1) >= Skv) v = -INFINITY;
    s[i] = v;
    mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float mn = fmaxf(m_run[r], mx[r]);
    alpha[r] = exp2_ftz(m_run[r] - mn);
    m_run[r] = mn;
    rs[r] = 0.f;
  }
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = (i >> 1) & 1;
    const float p0 = exp2_ftz(__fsub_rn(s[i], m_run[r])), p1 = exp2_ftz(__fsub_rn(s[i + 1], m_run[r]));
    rs[r] += p0 + p1;
    pa[i >> 3][(i & 7) >> 1] = pack_bf16x2(p0, p1);
  }
}

// KB 64-column blocks of head columns; NV = 40 (KB = 1, d <= 40) multiplies only what the head needs, as
// the backward does: S contracts over 3 k-steps (48 columns, the zeroed ones past d included) and O holds
// 40 columns, bitwise the results of the 64-column products.
template <int KB, int NV>
__global__ void __launch_bounds__(kAwThreads, 1) attn_fwd_wg_kernel(const __grid_constant__ AttnWgParams p) {
  static_assert(NV == 64 || (KB == 1 && NV == 40), "trimmed products only for one 64-column block");
  constexpr int KS = (NV + 15) / 16;   // k-steps of S per 64-column block
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  // [Q: 2 warpgroups x KB tiles][K: stages x KB][V: stages x KB]
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + 2 * KB * kTile;
  uint8_t* sV = sK + kAwStages * KB * kTile;
  __shared__ __align__(8) uint64_t q_bar;
  __shared__ __align__(8) uint64_t full_bar[kAwStages];
  __shared__ __align__(8) uint64_t empty_bar[kAwStages];

  const int wg = threadIdx.x >> 7;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * 128;
  const int nblk = (p.Skv + 63) / 64;
  constexpr uint32_t kv_bytes = 2 * KB * kTile;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.q_map);
    tma_prefetch_desc(&p.k_map);
    tma_prefetch_desc(&p.v_map);
    mbar_init(&q_bar, 1);
    for (int i = 0; i < kAwStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_sync();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&q_bar, 2 * KB * kTile);
      for (int w = 0; w < 2; ++w)
        for (int kb = 0; kb < KB; ++kb)
          tma_load_3d(sQ + (w * KB + kb) * kTile, &p.q_map, &q_bar, h * p.D + kb * 64, q0 + 64 * w, b);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % kAwStages;
        mbar_wait(&empty_bar[st], ((j / kAwStages) & 1) ^ 1);
        mbar_arrive_expect_tx(&full_bar[st], kv_bytes);
        for (int kb = 0; kb < KB; ++kb) {
          tma_load_3d(sK + (st * KB + kb) * kTile, &p.k_map, &full_bar[st], h * p.D + kb * 64, j * 64, b);
          tma_load_3d(sV + (st * KB + kb) * kTile, &p.v_map, &full_bar[st], h * p.D + kb * 64, j * 64, b);
        }
      }
    }
    return;
  }

  const int cw = wg - 1, et = threadIdx.x & 127, warp = et >> 5, lane = et & 31;
  uint8_t* myQ = sQ + cw * KB * kTile;
  mbar_wait(&q_bar, 0);
  // zero the Q columns past d (16-byte chunks of the swizzled tiles; d is a multiple of 8)
  if (p.D < KB * 64) {
    const int c0 = p.D >> 3, nch = KB * 8;
    for (int i = et; i < 64 * nch; i += 128) {
      const int row = i / nch, ch = i - row * nch;
      if (ch < c0) continue;
      const uint32_t a = smem_u32(myQ + (ch >> 3) * kTile) + row * 128 + (((ch & 7) ^ (row & 7)) << 4);
      sts128(a, 0u, 0u, 0u, 0u);
    }
    fence_proxy_async();   // generic-proxy writes before the wgmma (async proxy) reads
  }
  asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");

  float o[KB][NV / 2];
#pragma unroll
  for (int kb = 0; kb < KB; ++kb)
#pragma unroll
    for (int i = 0; i < NV / 2; ++i) o[kb][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(myQ);

  // one 64-key block; MASK only for the last block of a ragged Skv (the keys past Skv read as zero rows)
  auto block = [&](int j, auto mask) {
    const int st = j % kAwStages;
    mbar_wait(&full_bar[st], (j / kAwStages) & 1);
    const uint32_t k_addr = smem_u32(sK + st * KB * kTile);
    const uint32_t v_addr = smem_u32(sV + st * KB * kTile);
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb)
#pragma unroll
      for (int k = 0; k < KS; ++k)
        Wgmma<64, 0, 0>::mma(s, wgmma_desc_sw128(q_addr + kb * kTile + k * 32, 16, 1024),
                             wgmma_desc_sw128(k_addr + kb * kTile + k * 32, 16, 1024), (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);

    float alpha[2], rs[2];
    uint32_t pa[4][4];
    fwd_softmax<decltype(mask)::value>(s, m_run, alpha, rs, pa, p.c, j * 64 + 2 * (lane & 3), p.Skv);
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = __fmaf_rn(l_run[r], alpha[r], rs[r]);
    // alpha = 1 where the row maximum did not change: when it holds for every row of the warp, the
    // rescale (an exact multiply by 1) is skipped
    if (!__all_sync(0xffffffffu, alpha[0] == 1.f && alpha[1] == 1.f)) {
#pragma unroll
      for (int kb = 0; kb < KB; ++kb)
#pragma unroll
        for (int i = 0; i < NV / 2; ++i) o[kb][i] *= alpha[(i >> 1) & 1];
    }

    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int kb = 0; kb < KB; ++kb)   // V: 16 keys x NV head columns, MN-major
        WgmmaRs<NV, 1>::mma(o[kb], pa[kk], wgmma_desc_sw128(v_addr + kb * kTile + kk * 2048, kTile, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) wgmma_fence_acc(o[kb]);
    __syncwarp();
    if (et == 0) mbar_arrive(&empty_bar[st]);
  };
  const int nfull = p.Skv / 64;
  for (int j = 0; j < nfull; ++j) block(j, std::false_type());
  if (nfull < nblk) block(nfull, std::true_type());

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int row0 = q0 + 64 * cw + 16 * warp + (lane >> 2);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + 8 * r;
    if (row >= p.Sq) continue;
    const float inv = 1.f / l_run[r];
    bf16* orow = p.out + (static_cast<long long>(b) * p.Sq + row) * p.ldo + h * p.D;
#pragma unroll
    for (int kb = 0; kb < KB; ++kb)
#pragma unroll
      for (int q = 0; q < NV / 8; ++q) {
        const int col = kb * 64 + 8 * q + 2 * (lane & 3);
        if (col < p.D)
          *reinterpret_cast<uint32_t*>(orow + col) =
              pack_bf16x2(o[kb][4 * q + 2 * r] * inv, o[kb][4 * q + 2 * r + 1] * inv);
      }
    if ((lane & 3) == 0 && p.lse) p.lse[(static_cast<long long>(b) * p.H + h) * p.Sq + row] = m_run[r] + log2f(l_run[r]);
  }
}

// ------------------------------------------------------------------------------------------
// Backward, d <= 64 (one 64-column block).  One kernel body, two roles:
//   KV = true  (dK / dV): a consumer warpgroup keeps 64 keys of K and V resident and streams 64-query
//              tiles of Q and dO:  S^T = K Q^T, dP^T = V dO^T, P^T = exp2(c S^T - L[q]),
//              dS^T = P^T (dP^T - delta[q]);  dV += P^T dO, dK += dS^T Q  (dK scaled at the end).
//   KV = false (dQ): it keeps 64 queries of Q and dO resident and streams 64-key tiles of K and V:
//              S = Q K^T, dP = dO V^T, dS = P (dP - delta);  dQ += dS K.
// S and dP are SS-form wgmma; P^T / dS (bf16, packed from the accumulator fragment) are the register
// A operand of the RS-form wgmma against the streamed tile read MN-major, as in the forward.  The
// columns past d of the resident tiles are zeroed, so the next head's columns that the 64-wide boxes
// also cover add nothing; keys past Skv are masked, queries past Sq have L = +inf (P = 0).
// For d <= 40 only what the head needs is multiplied: S and dP contract over 3 k-steps (48 columns, the
// zeroed ones past d included) and the accumulators hold 40 columns (NV = 40).  The dropped k-step only
// added products with zeroed columns and the dropped columns were never stored, so the results are
// those of the 64-column products bit for bit.
// Pipeline: block j's S / dP products are issued ahead of block j-1's accumulator products, and block
// j's elementwise P / dS work runs while the latter are on the tensor cores.
// ------------------------------------------------------------------------------------------
struct alignas(64) AttnBwdParams {
  CUtensorMap fix0_map, fix1_map;   // resident tiles: K, V (KV) or Q, dO
  CUtensorMap str0_map, str1_map;   // streamed tiles: Q, dO (KV) or K, V
  const float *lse, *delta;
  bf16 *out0, *out1;                // KV: dK, dV;  dQ: dQ (out1 unused)
  long long ld0, ld1;
  int H, Sq, Skv, D;
  int n_fix, n_str;                 // rows of the resident / streamed sequences
  float c, scale;
};

// P and dS of one 64-column block, in place: s becomes P, dp becomes dS (fp32).  KV: row = key (valid
// per row), the column statistics lc / dc were loaded for this block; dQ: column = key, MASK when the
// block's keys from kcol on may lie past Skv.  c S - L is one FFMA, as the expression always compiled to.
template <bool KV, bool MASK>
__device__ __forceinline__ void bwd_elementwise(float (&s)[32], float (&dp)[32], const float (&lc)[16],
                                                const float (&dc)[16], const float (&lrow)[2],
                                                const float (&drow)[2], const bool (&rvalid)[2], float c,
                                                int kcol, int Skv) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = (i >> 1) & 1;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float l, d;
      bool ok;
      if (KV) {
        l = lc[2 * (i >> 2) + e];
        d = dc[2 * (i >> 2) + e];
        ok = rvalid[r];
      } else {
        l = lrow[r];
        d = drow[r];
        ok = !MASK || kcol + 8 * (i >> 2) + e < Skv;
      }
      const float pv = ok ? exp2_ftz(__fmaf_rn(s[i + e], c, -l)) : 0.f;
      s[i + e] = pv;
      dp[i + e] = pv * (dp[i + e] - d);
    }
  }
}

template <bool KV, int NV>
__global__ void __launch_bounds__(kAwThreads, 1) attn_bwd_wg_kernel(const __grid_constant__ AttnBwdParams p) {
  constexpr int kStages = kBwdStages;
  constexpr int KS = (NV + 15) / 16;   // k-steps of S / dP
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sF = smem;                          // [2 warpgroups][2 tiles]
  uint8_t* sS = sF + 4 * kTile;                // [stages][2 tiles]
  __shared__ __align__(8) uint64_t f_bar;
  __shared__ __align__(8) uint64_t full_bar[kStages];
  __shared__ __align__(8) uint64_t empty_bar[kStages];
  // (KV) L and delta of the streamed query block, per consumer warpgroup, double-buffered
  __shared__ float stats[2][2][2][64];   // [warpgroup][buffer][L, delta][query]

  const int wg = threadIdx.x >> 7;
  const int b = blockIdx.z, h = blockIdx.y, r0 = blockIdx.x * 128;
  const int nblk = (p.n_str + 63) / 64;
  const int col0 = h * p.D;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.fix0_map);
    tma_prefetch_desc(&p.fix1_map);
    tma_prefetch_desc(&p.str0_map);
    tma_prefetch_desc(&p.str1_map);
    mbar_init(&f_bar, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_sync();

  if (wg == 0) {
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&f_bar, 4 * kTile);
      for (int w = 0; w < 2; ++w) {
        tma_load_3d(sF + (2 * w) * kTile, &p.fix0_map, &f_bar, col0, r0 + 64 * w, b);
        tma_load_3d(sF + (2 * w + 1) * kTile, &p.fix1_map, &f_bar, col0, r0 + 64 * w, b);
      }
      for (int j = 0; j < nblk; ++j) {
        const int st = j % kStages;
        mbar_wait(&empty_bar[st], ((j / kStages) & 1) ^ 1);
        mbar_arrive_expect_tx(&full_bar[st], 2 * kTile);
        tma_load_3d(sS + (2 * st) * kTile, &p.str0_map, &full_bar[st], col0, j * 64, b);
        tma_load_3d(sS + (2 * st + 1) * kTile, &p.str1_map, &full_bar[st], col0, j * 64, b);
      }
    }
    return;
  }

  regs_alloc<232>();
  const int cw = wg - 1, et = threadIdx.x & 127, warp = et >> 5, lane = et & 31;
  uint8_t* myF = sF + 2 * cw * kTile;
  mbar_wait(&f_bar, 0);
  if (p.D < 64) {   // zero the resident columns past d (both tiles)
    const int c0 = p.D >> 3;
    for (int i = et; i < 2 * 64 * 8; i += 128) {
      const int t = i >> 9, row = (i >> 3) & 63, ch = i & 7;
      if (ch < c0) continue;
      sts128(smem_u32(myF + t * kTile) + row * 128 + ((ch ^ (row & 7)) << 4), 0u, 0u, 0u, 0u);
    }
    fence_proxy_async();
  }
  asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");

  const float* L = p.lse + (static_cast<long long>(b) * p.H + h) * p.Sq;
  const float* Dl = p.delta + (static_cast<long long>(b) * p.H + h) * p.Sq;
  // accumulator fragment rows of this thread: r0 + 64 cw + 16 warp + lane / 4 (+8)
  const int frow = r0 + 64 * cw + 16 * warp + (lane >> 2);
  float lrow[2] = {0.f, 0.f}, drow[2] = {0.f, 0.f};
  bool rvalid[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    rvalid[r] = frow + 8 * r < p.n_fix;
    if (!KV) {
      lrow[r] = rvalid[r] ? L[frow + 8 * r] : INFINITY;
      drow[r] = rvalid[r] ? Dl[frow + 8 * r] : 0.f;
    }
  }
  float acc0[NV / 2], acc1[NV / 2];   // KV: dK, dV;  dQ: dQ (acc1 unused)
#pragma unroll
  for (int i = 0; i < NV / 2; ++i) acc0[i] = acc1[i] = 0.f;
  const uint32_t f0 = smem_u32(myF), f1 = f0 + kTile;
  const bool ragged = !KV && (p.Skv & 63) != 0;
  float s[32], dp[32];
  uint32_t pa[4][4], dsa[4][4];         // P^T / dS of the previous block as register A operands

  auto issue_sdp = [&](int st) {
    const uint32_t s0 = smem_u32(sS + 2 * st * kTile), s1 = s0 + kTile;
    Wgmma<64, 0, 0>::mma_first(s, wgmma_desc_sw128(f0, 16, 1024), wgmma_desc_sw128(s0, 16, 1024));
    Wgmma<64, 0, 0>::mma_first(dp, wgmma_desc_sw128(f1, 16, 1024), wgmma_desc_sw128(s1, 16, 1024));
#pragma unroll
    for (int k = 1; k < KS; ++k) {
      Wgmma<64, 0, 0>::mma(s, wgmma_desc_sw128(f0 + k * 32, 16, 1024), wgmma_desc_sw128(s0 + k * 32, 16, 1024), 1u);
      Wgmma<64, 0, 0>::mma(dp, wgmma_desc_sw128(f1 + k * 32, 16, 1024), wgmma_desc_sw128(s1 + k * 32, 16, 1024), 1u);
    }
    wgmma_commit();
  };
  auto issue_acc = [&](int st) {
    const uint32_t s0 = smem_u32(sS + 2 * st * kTile), s1 = s0 + kTile;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // streamed tile 0 (Q for dK, K for dQ) and 1 (dO for dV), 16 rows x NV columns, MN-major
      WgmmaRs<NV, 1>::mma(acc0, dsa[kk], wgmma_desc_sw128(s0 + kk * 2048, kTile, 1024), 1u);
      if (KV) WgmmaRs<NV, 1>::mma(acc1, pa[kk], wgmma_desc_sw128(s1 + kk * 2048, kTile, 1024), 1u);
    }
    wgmma_commit();
  };
  // (KV) the L / delta of query block j: one value per thread, loaded a block ahead of its use (the
  // load runs under the block's MMAs and elementwise work), published through shared memory
  auto load_stat = [&](int j) {
    const int qi = j * 64 + (et & 63);
    if (et < 64) return qi < p.Sq ? L[qi] : INFINITY;
    return qi < p.Sq ? Dl[qi] : 0.f;
  };
  auto publish_stat = [&](int j, float v) {
    stats[cw][j & 1][et >> 6][et & 63] = v;
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
  };
  auto elementwise = [&](int j) {
    const int kcol = j * 64 + 2 * (lane & 3);
    float lc[16], dc[16];   // (KV) statistics of the block's 16 query columns of the thread
    if (KV) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float2 l2 = *reinterpret_cast<const float2*>(&stats[cw][j & 1][0][8 * q + 2 * (lane & 3)]);
        const float2 d2 = *reinterpret_cast<const float2*>(&stats[cw][j & 1][1][8 * q + 2 * (lane & 3)]);
        lc[2 * q] = l2.x;
        lc[2 * q + 1] = l2.y;
        dc[2 * q] = d2.x;
        dc[2 * q + 1] = d2.y;
      }
    }
    if (ragged && j == nblk - 1)
      bwd_elementwise<KV, true>(s, dp, lc, dc, lrow, drow, rvalid, p.c, kcol, p.Skv);
    else
      bwd_elementwise<KV, false>(s, dp, lc, dc, lrow, drow, rvalid, p.c, kcol, p.Skv);
  };

  if (KV) publish_stat(0, load_stat(0));
  mbar_wait(&full_bar[0], 0);
  wgmma_fence();
  issue_sdp(0);
  float nxt = KV ? load_stat(1) : 0.f;
  wgmma_wait<0>();
  wgmma_fence_acc(s);
  wgmma_fence_acc(dp);
  elementwise(0);
  if (KV) publish_stat(1, nxt);
  pack_operand(pa, s);
  pack_operand(dsa, dp);

  for (int j = 1; j < nblk; ++j) {
    const int st = j % kStages, pst = (j - 1) % kStages;
    mbar_wait(&full_bar[st], (j / kStages) & 1);
    wgmma_fence();
    issue_sdp(st);       // S_j, dP_j ...
    issue_acc(pst);      // ... then the accumulator products of block j-1
    if (KV) nxt = load_stat(j + 1);
    wgmma_wait<1>();     // S_j and dP_j have landed
    wgmma_fence_acc(s);
    wgmma_fence_acc(dp);
    elementwise(j);
    if (KV) publish_stat(j + 1, nxt);
    wgmma_wait<0>();
    wgmma_fence_acc(acc0);
    wgmma_fence_acc(acc1);
    keep_operand(pa);
    keep_operand(dsa);
    __syncwarp();
    if (et == 0) mbar_arrive(&empty_bar[pst]);
    pack_operand(pa, s);
    pack_operand(dsa, dp);
  }
  wgmma_fence();
  issue_acc((nblk - 1) % kStages);
  wgmma_wait<0>();
  wgmma_fence_acc(acc0);
  wgmma_fence_acc(acc1);
  keep_operand(pa);
  keep_operand(dsa);

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!rvalid[r]) continue;
    const long long row = static_cast<long long>(b) * p.n_fix + frow + 8 * r;
    bf16* o0 = p.out0 + row * p.ld0 + col0;
    bf16* o1 = KV ? p.out1 + row * p.ld1 + col0 : nullptr;
#pragma unroll
    for (int q = 0; q < NV / 8; ++q) {
      const int col = 8 * q + 2 * (lane & 3);
      if (col < p.D) {
        *reinterpret_cast<uint32_t*>(o0 + col) =
            pack_bf16x2(acc0[4 * q + 2 * r] * p.scale, acc0[4 * q + 2 * r + 1] * p.scale);
        if (KV) *reinterpret_cast<uint32_t*>(o1 + col) = pack_bf16x2(acc1[4 * q + 2 * r], acc1[4 * q + 2 * r + 1]);
      }
    }
  }
}

// 3-D map (head columns, sequence, batch) with 64 x 64 SWIZZLE_128B boxes; rows past S and columns
// past H*D read as zero.  pcm_attn_fwd / pcm_attn_bwd have already checked that the base is 16-byte
// aligned and ld a multiple of 8, as TMA requires.
int encode_seq_map(CUtensorMap* m, const void* base, int HD, int S, int B, long long ld) {
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld & 7) != 0)
    return set_error("attention: tensor map base not 16-byte aligned or row stride not a multiple of 8");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(HD), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(B)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld) * 2, static_cast<cuuint64_t>(ld) * 2 * S};
  cuuint32_t box[3] = {64, 64, 1}, estr[3] = {1, 1, 1};
  return encode_tmap(m, base, 3, dims, strides, box, estr);
}

template <int KB, int NV>
cudaError_t launch_fwd(dim3 grid, cudaStream_t stream, const AttnWgParams& p) {
  const size_t smem = KB * (2 + 2 * kAwStages) * kTile + 1024;
  static bool attr = false;
  if (!attr) {
    const cudaError_t e = cudaFuncSetAttribute(attn_fwd_wg_kernel<KB, NV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return launch_pdl(attn_fwd_wg_kernel<KB, NV>, grid, dim3(kAwThreads), smem, stream, p);
}

template <bool KV, int NV>
cudaError_t launch_bwd(dim3 grid, cudaStream_t stream, const AttnBwdParams& p) {
  const size_t smem = (4 + 2 * kBwdStages) * kTile + 1024;
  static bool attr = false;
  if (!attr) {
    const cudaError_t e = cudaFuncSetAttribute(attn_bwd_wg_kernel<KV, NV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return launch_pdl(attn_bwd_wg_kernel<KV, NV>, grid, dim3(kAwThreads), smem, stream, p);
}

}  // namespace

// Returns 0 on launch, < 0 on error, 1 for d > 128 (the caller runs attn.cu's kernel).
int attn_fwd_wg(const void* q, const void* k, const void* v, void* out, float* lse, int B, int H, int Sq,
                int Skv, int D, long long ldq, long long ldk, long long ldv, long long ldo, float scale,
                cudaStream_t stream) {
  if (D % 8 != 0 || D > 128) return 1;
  static AttnWgParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  if ((rc = encode_seq_map(&p.q_map, q, H * D, Sq, B, ldq)) != 0) return rc;
  if ((rc = encode_seq_map(&p.k_map, k, H * D, Skv, B, ldk)) != 0) return rc;
  if ((rc = encode_seq_map(&p.v_map, v, H * D, Skv, B, ldv)) != 0) return rc;
  p.out = reinterpret_cast<bf16*>(out);
  p.lse = lse;
  p.H = H; p.Sq = Sq; p.Skv = Skv; p.D = D; p.ldo = ldo;
  p.c = scale * 1.4426950408889634f;
  const dim3 grid((Sq + 127) / 128, H, B);
  if (D <= 40)
    CUDA_TRY((launch_fwd<1, 40>)(grid, stream, p));
  else if (D <= 64)
    CUDA_TRY((launch_fwd<1, 64>)(grid, stream, p));
  else
    CUDA_TRY((launch_fwd<2, 64>)(grid, stream, p));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// dK, dV and dQ from q, k, v, dO and the forward's lse plus delta = rowsum(dO o O) (already computed).
// Returns 0 on launch, < 0 on error, 1 for d > 64 (the caller runs attn.cu's kernels).
int attn_bwd_wg(const void* q, const void* k, const void* v, const void* dout, const float* lse,
                const float* delta, void* dq, void* dk, void* dv, int B, int H, int Sq, int Skv, int D,
                long long ldq, long long ldk, long long ldv, long long ldo, float scale, cudaStream_t stream) {
  if (D % 8 != 0 || D > 64) return 1;
  static AttnBwdParams pk, pq;
  memset(&pk, 0, sizeof(pk));
  int rc;
  if ((rc = encode_seq_map(&pk.fix0_map, k, H * D, Skv, B, ldk)) != 0) return rc;
  if ((rc = encode_seq_map(&pk.fix1_map, v, H * D, Skv, B, ldv)) != 0) return rc;
  if ((rc = encode_seq_map(&pk.str0_map, q, H * D, Sq, B, ldq)) != 0) return rc;
  if ((rc = encode_seq_map(&pk.str1_map, dout, H * D, Sq, B, ldo)) != 0) return rc;
  pk.lse = lse; pk.delta = delta;
  pk.H = H; pk.Sq = Sq; pk.Skv = Skv; pk.D = D;
  pk.c = scale * 1.4426950408889634f;
  pq = pk;
  // dK / dV: resident K, V (rows = keys), streamed Q, dO
  pk.out0 = reinterpret_cast<bf16*>(dk); pk.ld0 = ldk;
  pk.out1 = reinterpret_cast<bf16*>(dv); pk.ld1 = ldv;
  pk.n_fix = Skv; pk.n_str = Sq; pk.scale = scale;
  // dQ: resident Q, dO (rows = queries), streamed K, V
  pq.fix0_map = pk.str0_map; pq.fix1_map = pk.str1_map;
  pq.str0_map = pk.fix0_map; pq.str1_map = pk.fix1_map;
  pq.out0 = reinterpret_cast<bf16*>(dq); pq.ld0 = ldq;
  pq.out1 = nullptr; pq.ld1 = 0;
  pq.n_fix = Sq; pq.n_str = Skv; pq.scale = scale;
  const dim3 gk((Skv + 127) / 128, H, B), gq((Sq + 127) / 128, H, B);
  if (D <= 40) {
    CUDA_TRY((launch_bwd<true, 40>)(gk, stream, pk));
    CUDA_TRY((launch_bwd<false, 40>)(gq, stream, pq));
  } else {
    CUDA_TRY((launch_bwd<true, 64>)(gk, stream, pk));
    CUDA_TRY((launch_bwd<false, 64>)(gq, stream, pq));
  }
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace pcm
