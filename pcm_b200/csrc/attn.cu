// Flash-style self / cross attention, forward and backward, for the SD1.5 UNet head sizes
// (8 heads, d = 40 / 80 / 160; kv = tokens or 77 text tokens).  No S x S matrix is materialised.
// Warp-level mma.sync.m16n8k16 bf16 tensor-core path with cp.async double-buffered K/V tiles, for the
// head sizes the wgmma / TMA kernels (attn_wg.cu) do not cover: forward d = 160, backward d > 64.
//
// Replaces xformers / torch SDPA attention inside diffusers' Attention processor
// (enabled at train_pcm_lora_sd15.py:947-961; called from the UNet forwards at :1192-1198,
// 1219-1244, 1263-1268) and its backward (:1296).
//
// Layout: q [B, Sq, H*D] (row stride ldq), k / v [B, Skv, H*D] (ldk / ldv), o like q;
// lse, delta [B, H, Sq] fp32 (lse in log2 units of the scaled scores).
#include <stdlib.h>
#include "common.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"

namespace pcm {

struct AttnParams {
  const bf16 *q, *k, *v, *o, *dout;
  bf16 *out, *dq, *dk, *dv;
  float *lse, *delta;
  int B, H, Sq, Skv, D;
  long long ldq, ldk, ldv, ldo;
  float scale;
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragment (16 rows x 16 k) from row-major [row][k] smem
template <int LDS>
__device__ __forceinline__ void load_a(uint32_t (&a)[4], const bf16* s, int row0, int k0, int lane) {
  ldsm_x4(a, s + (row0 + (lane & 15)) * LDS + k0 + (lane >> 4) * 8);
}
// B fragments for two n-tiles (16 n x 16 k) from row-major [n][k] smem: r0,r1 -> n-tile 0
template <int LDS>
__device__ __forceinline__ void load_b_nk(uint32_t (&r)[4], const bf16* s, int n0, int k0, int lane) {
  ldsm_x4(r, s + (n0 + (lane & 7) + (lane >> 4) * 8) * LDS + k0 + ((lane >> 3) & 1) * 8);
}
// B fragments for two n-tiles (16 k x 16 n) from row-major [k][n] smem (transposed load)
template <int LDS>
__device__ __forceinline__ void load_b_kn(uint32_t (&r)[4], const bf16* s, int k0, int n0, int lane) {
  ldsm_x4_t(r, s + (k0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + n0 + (lane >> 4) * 8);
}

// async copy of a [rows x DP] tile (DP/8 16-byte chunks per row; chunks >= D and rows >= limit are
// zero filled) from a [*, ld] global matrix into [rows][LDS] shared memory
template <int DP, int LDS, int ROWS, int THREADS>
__device__ __forceinline__ void load_tile(bf16* s, const bf16* g, long long ld, int row0, int limit,
                                          int D, int tid) {
  constexpr int CH = DP / 8;
  for (int i = tid; i < ROWS * CH; i += THREADS) {
    const int r = i / CH, c = i - r * CH;
    bf16* dst = s + r * LDS + c * 8;
    if (row0 + r < limit && c * 8 < D)
      cp_async16(dst, g + static_cast<long long>(row0 + r) * ld + c * 8);
    else
      *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
  }
}

constexpr float kLog2e = 1.4426950408889634f;

// ------------------------------------------------------------------------------------------
// forward: 128 query rows per CTA (8 warps x 16 rows), 64-key tiles
// ------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(256) attn_fwd_kernel(const AttnParams p) {
  griddep_sync();
  constexpr int LDS = DP + 8, BM = 128, BN = 64, T = 256;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  bf16* sQ = reinterpret_cast<bf16*>(smem_attn);
  bf16* sK = sQ + BM * LDS;
  bf16* sV = sK + 2 * BN * LDS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BM;
  const bf16* Q = p.q + static_cast<long long>(b) * p.Sq * p.ldq + h * p.D;
  const bf16* K = p.k + static_cast<long long>(b) * p.Skv * p.ldk + h * p.D;
  const bf16* V = p.v + static_cast<long long>(b) * p.Skv * p.ldv + h * p.D;
  const int nblk = (p.Skv + BN - 1) / BN;
  const float c = p.scale * kLog2e;

  load_tile<DP, LDS, BM, T>(sQ, Q, p.ldq, q0, p.Sq, p.D, tid);
  load_tile<DP, LDS, BN, T>(sK, K, p.ldk, 0, p.Skv, p.D, tid);
  load_tile<DP, LDS, BN, T>(sV, V, p.ldv, 0, p.Skv, p.D, tid);
  cp_async_commit();

  float oacc[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  for (int j = 0; j < nblk; ++j) {
    const int st = j & 1;
    if (j + 1 < nblk) {
      load_tile<DP, LDS, BN, T>(sK + (st ^ 1) * BN * LDS, K, p.ldk, (j + 1) * BN, p.Skv, p.D, tid);
      load_tile<DP, LDS, BN, T>(sV + (st ^ 1) * BN * LDS, V, p.ldv, (j + 1) * BN, p.Skv, p.D, tid);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* sKs = sK + st * BN * LDS;
    const bf16* sVs = sV + st * BN * LDS;

    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
      uint32_t a[4];
      load_a<LDS>(a, sQ, warp * 16, kk * 16, lane);
#pragma unroll
      for (int n2 = 0; n2 < 4; ++n2) {
        uint32_t r[4];
        load_b_nk<LDS>(r, sKs, n2 * 16, kk * 16, lane);
        mma16816(s[2 * n2], a, r[0], r[1]);
        mma16816(s[2 * n2 + 1], a, r[2], r[3]);
      }
    }
    // scale, mask, online softmax
    const int kbase = j * BN + (lane & 3) * 2;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + i * 8 + (e & 1);
        const float v = key < p.Skv ? s[i][e] * c : -INFINITY;
        s[i][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m_run[r], mx[r]);
      alpha[r] = exp2f(m_run[r] - mn);
      m_run[r] = mn;
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pa[4][4];  // P as A fragments for 4 k-steps of 16 keys
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float p0 = exp2f(s[i][0] - m_run[0]), p1 = exp2f(s[i][1] - m_run[0]);
      const float p2 = exp2f(s[i][2] - m_run[1]), p3 = exp2f(s[i][3] - m_run[1]);
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      pa[i >> 1][(i & 1) * 2] = pack_bf16x2(p0, p1);
      pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + rs[r];
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      oacc[i][0] *= alpha[0];
      oacc[i][1] *= alpha[0];
      oacc[i][2] *= alpha[1];
      oacc[i][3] *= alpha[1];
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int d2 = 0; d2 < DP / 16; ++d2) {
        uint32_t r[4];
        load_b_kn<LDS>(r, sVs, kk * 16, d2 * 16, lane);
        mma16816(oacc[2 * d2], pa[kk], r[0], r[1]);
        mma16816(oacc[2 * d2 + 1], pa[kk], r[2], r[3]);
      }
    }
    __syncthreads();
  }
  // finalize
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int row0 = q0 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + r * 8;
    if (row >= p.Sq) continue;
    const float inv = 1.f / l_run[r];
    bf16* orow = p.out + (static_cast<long long>(b) * p.Sq + row) * p.ldo + h * p.D;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      const int col = i * 8 + (lane & 3) * 2;
      if (col < p.D)
        *reinterpret_cast<uint32_t*>(orow + col) =
            pack_bf16x2(oacc[i][2 * r] * inv, oacc[i][2 * r + 1] * inv);
    }
    if ((lane & 3) == 0 && p.lse)
      p.lse[(static_cast<long long>(b) * p.H + h) * p.Sq + row] = m_run[r] + log2f(l_run[r]);
  }
}

// delta[b,h,s] = sum_d dO * O
__global__ void attn_delta_kernel(const AttnParams p) {
  griddep_sync();
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long total = static_cast<long long>(p.B) * p.Sq * p.H;
  if (i >= total) return;
  const int h = static_cast<int>(i % p.H);
  const long long bs = i / p.H;
  const int s = static_cast<int>(bs % p.Sq);
  const int b = static_cast<int>(bs / p.Sq);
  const bf16* o = p.o + bs * p.ldo + h * p.D;
  const bf16* d = p.dout + bs * p.ldo + h * p.D;
  float acc = 0.f;
  for (int c = 0; c < p.D; c += 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(o + c);
    const uint4 w = *reinterpret_cast<const uint4*>(d + c);
    const uint32_t uu[4] = {u.x, u.y, u.z, u.w}, ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = unpack_bf16x2(uu[k]), bb = unpack_bf16x2(ww[k]);
      acc += a.x * bb.x + a.y * bb.y;
    }
  }
  p.delta[(static_cast<long long>(b) * p.H + h) * p.Sq + s] = acc;
}

// ------------------------------------------------------------------------------------------
// backward 1: dK, dV.  64 keys per CTA (4 warps x 16 keys), loop over 64-query tiles.
// Works on transposed score tiles  S^T = K Q^T  so P^T / dS^T feed the second GEMMs directly.
// ------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(128) attn_bwd_dkdv_kernel(const AttnParams p) {
  griddep_sync();
  constexpr int LDS = DP + 8, BQ = 64, BN = 64, T = 128;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  bf16* sK = reinterpret_cast<bf16*>(smem_attn);
  bf16* sV = sK + BN * LDS;
  bf16* sQ = sV + BN * LDS;        // [2][BQ][LDS]
  bf16* sdO = sQ + 2 * BQ * LDS;   // [2][BQ][LDS]
  float* sL = reinterpret_cast<float*>(sdO + 2 * BQ * LDS);  // [2][BQ]
  float* sD = sL + 2 * BQ;                                   // [2][BQ]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, n0 = blockIdx.x * BN;
  const bf16* Q = p.q + static_cast<long long>(b) * p.Sq * p.ldq + h * p.D;
  const bf16* dO = p.dout + static_cast<long long>(b) * p.Sq * p.ldo + h * p.D;
  const bf16* K = p.k + static_cast<long long>(b) * p.Skv * p.ldk + h * p.D;
  const bf16* V = p.v + static_cast<long long>(b) * p.Skv * p.ldv + h * p.D;
  const float* L = p.lse + (static_cast<long long>(b) * p.H + h) * p.Sq;
  const float* Dl = p.delta + (static_cast<long long>(b) * p.H + h) * p.Sq;
  const int nqb = (p.Sq + BQ - 1) / BQ;
  const float c = p.scale * kLog2e;

  auto load_q_tiles = [&](int st, int qb) {
    load_tile<DP, LDS, BQ, T>(sQ + st * BQ * LDS, Q, p.ldq, qb * BQ, p.Sq, p.D, tid);
    load_tile<DP, LDS, BQ, T>(sdO + st * BQ * LDS, dO, p.ldo, qb * BQ, p.Sq, p.D, tid);
    if (tid < BQ) {
      const int row = qb * BQ + tid;
      sL[st * BQ + tid] = row < p.Sq ? L[row] : INFINITY;
      sD[st * BQ + tid] = row < p.Sq ? Dl[row] : 0.f;
    }
  };
  load_tile<DP, LDS, BN, T>(sK, K, p.ldk, n0, p.Skv, p.D, tid);
  load_tile<DP, LDS, BN, T>(sV, V, p.ldv, n0, p.Skv, p.D, tid);
  load_q_tiles(0, 0);
  cp_async_commit();

  float dk[DP / 8][4], dv[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }
  const int key0 = n0 + warp * 16 + (lane >> 2);
  const bool kvalid[2] = {key0 < p.Skv, key0 + 8 < p.Skv};

  for (int qb = 0; qb < nqb; ++qb) {
    const int st = qb & 1;
    if (qb + 1 < nqb) load_q_tiles(st ^ 1, qb + 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* sQs = sQ + st * BQ * LDS;
    const bf16* sdOs = sdO + st * BQ * LDS;
    const float* sLs = sL + st * BQ;
    const float* sDs = sD + st * BQ;

    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
      uint32_t ak[4], av[4];
      load_a<LDS>(ak, sK, warp * 16, kk * 16, lane);
      load_a<LDS>(av, sV, warp * 16, kk * 16, lane);
#pragma unroll
      for (int n2 = 0; n2 < 4; ++n2) {
        uint32_t r[4];
        load_b_nk<LDS>(r, sQs, n2 * 16, kk * 16, lane);
        mma16816(s[2 * n2], ak, r[0], r[1]);
        mma16816(s[2 * n2 + 1], ak, r[2], r[3]);
        load_b_nk<LDS>(r, sdOs, n2 * 16, kk * 16, lane);
        mma16816(dp[2 * n2], av, r[0], r[1]);
        mma16816(dp[2 * n2 + 1], av, r[2], r[3]);
      }
    }
    // P^T and dS^T -> A fragments (k = query index)
    uint32_t pa[4][4], dsa[4][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int qc = i * 8 + (lane & 3) * 2;
      const float l0 = sLs[qc], l1 = sLs[qc + 1];
      const float d0 = sDs[qc], d1 = sDs[qc + 1];
      float pv[4];
      pv[0] = kvalid[0] ? exp2f(s[i][0] * c - l0) : 0.f;
      pv[1] = kvalid[0] ? exp2f(s[i][1] * c - l1) : 0.f;
      pv[2] = kvalid[1] ? exp2f(s[i][2] * c - l0) : 0.f;
      pv[3] = kvalid[1] ? exp2f(s[i][3] * c - l1) : 0.f;
      const float g0 = pv[0] * (dp[i][0] - d0), g1 = pv[1] * (dp[i][1] - d1);
      const float g2 = pv[2] * (dp[i][2] - d0), g3 = pv[3] * (dp[i][3] - d1);
      pa[i >> 1][(i & 1) * 2] = pack_bf16x2(pv[0], pv[1]);
      pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(pv[2], pv[3]);
      dsa[i >> 1][(i & 1) * 2] = pack_bf16x2(g0, g1);
      dsa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(g2, g3);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int d2 = 0; d2 < DP / 16; ++d2) {
        uint32_t r[4];
        load_b_kn<LDS>(r, sdOs, kk * 16, d2 * 16, lane);
        mma16816(dv[2 * d2], pa[kk], r[0], r[1]);
        mma16816(dv[2 * d2 + 1], pa[kk], r[2], r[3]);
        load_b_kn<LDS>(r, sQs, kk * 16, d2 * 16, lane);
        mma16816(dk[2 * d2], dsa[kk], r[0], r[1]);
        mma16816(dk[2 * d2 + 1], dsa[kk], r[2], r[3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key0 + r * 8;
    if (key >= p.Skv) continue;
    bf16* dkrow = p.dk + (static_cast<long long>(b) * p.Skv + key) * p.ldk + h * p.D;
    bf16* dvrow = p.dv + (static_cast<long long>(b) * p.Skv + key) * p.ldv + h * p.D;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      const int col = i * 8 + (lane & 3) * 2;
      if (col < p.D) {
        *reinterpret_cast<uint32_t*>(dkrow + col) =
            pack_bf16x2(dk[i][2 * r] * p.scale, dk[i][2 * r + 1] * p.scale);
        *reinterpret_cast<uint32_t*>(dvrow + col) = pack_bf16x2(dv[i][2 * r], dv[i][2 * r + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// backward 2: dQ.  64 queries per CTA (4 warps x 16 rows), loop over 64-key tiles.
// ------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const AttnParams p) {
  griddep_sync();
  constexpr int LDS = DP + 8, BQ = 64, BN = 64, T = 128;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  bf16* sQ = reinterpret_cast<bf16*>(smem_attn);
  bf16* sdO = sQ + BQ * LDS;
  bf16* sK = sdO + BQ * LDS;      // [2][BN][LDS]
  bf16* sV = sK + 2 * BN * LDS;   // [2][BN][LDS]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
  const bf16* Q = p.q + static_cast<long long>(b) * p.Sq * p.ldq + h * p.D;
  const bf16* dO = p.dout + static_cast<long long>(b) * p.Sq * p.ldo + h * p.D;
  const bf16* K = p.k + static_cast<long long>(b) * p.Skv * p.ldk + h * p.D;
  const bf16* V = p.v + static_cast<long long>(b) * p.Skv * p.ldv + h * p.D;
  const int nblk = (p.Skv + BN - 1) / BN;
  const float c = p.scale * kLog2e;

  load_tile<DP, LDS, BQ, T>(sQ, Q, p.ldq, q0, p.Sq, p.D, tid);
  load_tile<DP, LDS, BQ, T>(sdO, dO, p.ldo, q0, p.Sq, p.D, tid);
  load_tile<DP, LDS, BN, T>(sK, K, p.ldk, 0, p.Skv, p.D, tid);
  load_tile<DP, LDS, BN, T>(sV, V, p.ldv, 0, p.Skv, p.D, tid);
  cp_async_commit();

  const int row0 = q0 + warp * 16 + (lane >> 2);
  float lrow[2], drow[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + r * 8;
    const long long li = (static_cast<long long>(b) * p.H + h) * p.Sq + row;
    lrow[r] = row < p.Sq ? p.lse[li] : INFINITY;
    drow[r] = row < p.Sq ? p.delta[li] : 0.f;
  }
  float dq[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;

  for (int j = 0; j < nblk; ++j) {
    const int st = j & 1;
    if (j + 1 < nblk) {
      load_tile<DP, LDS, BN, T>(sK + (st ^ 1) * BN * LDS, K, p.ldk, (j + 1) * BN, p.Skv, p.D, tid);
      load_tile<DP, LDS, BN, T>(sV + (st ^ 1) * BN * LDS, V, p.ldv, (j + 1) * BN, p.Skv, p.D, tid);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* sKs = sK + st * BN * LDS;
    const bf16* sVs = sV + st * BN * LDS;
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
      uint32_t aq[4], ad[4];
      load_a<LDS>(aq, sQ, warp * 16, kk * 16, lane);
      load_a<LDS>(ad, sdO, warp * 16, kk * 16, lane);
#pragma unroll
      for (int n2 = 0; n2 < 4; ++n2) {
        uint32_t r[4];
        load_b_nk<LDS>(r, sKs, n2 * 16, kk * 16, lane);
        mma16816(s[2 * n2], aq, r[0], r[1]);
        mma16816(s[2 * n2 + 1], aq, r[2], r[3]);
        load_b_nk<LDS>(r, sVs, n2 * 16, kk * 16, lane);
        mma16816(dp[2 * n2], ad, r[0], r[1]);
        mma16816(dp[2 * n2 + 1], ad, r[2], r[3]);
      }
    }
    uint32_t dsa[4][4];
    const int kbase = j * BN + (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float g[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + i * 8 + (e & 1);
        const float pv = key < p.Skv ? exp2f(s[i][e] * c - lrow[e >> 1]) : 0.f;
        g[e] = pv * (dp[i][e] - drow[e >> 1]);
      }
      dsa[i >> 1][(i & 1) * 2] = pack_bf16x2(g[0], g[1]);
      dsa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(g[2], g[3]);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int d2 = 0; d2 < DP / 16; ++d2) {
        uint32_t r[4];
        load_b_kn<LDS>(r, sKs, kk * 16, d2 * 16, lane);
        mma16816(dq[2 * d2], dsa[kk], r[0], r[1]);
        mma16816(dq[2 * d2 + 1], dsa[kk], r[2], r[3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + r * 8;
    if (row >= p.Sq) continue;
    bf16* dqrow = p.dq + (static_cast<long long>(b) * p.Sq + row) * p.ldq + h * p.D;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      const int col = i * 8 + (lane & 3) * 2;
      if (col < p.D)
        *reinterpret_cast<uint32_t*>(dqrow + col) =
            pack_bf16x2(dq[i][2 * r] * p.scale, dq[i][2 * r + 1] * p.scale);
    }
  }
}

template <int DP>
static int launch_fwd(const AttnParams& p, cudaStream_t stream) {
  constexpr int LDS = DP + 8;
  const size_t smem = static_cast<size_t>(128 + 4 * 64) * LDS * sizeof(bf16);
  static bool set = false;
  if (!set) {
    CUDA_TRY(cudaFuncSetAttribute(attn_fwd_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem)));
    set = true;
  }
  dim3 grid((p.Sq + 127) / 128, p.H, p.B);
  CUDA_TRY(launch_pdl(attn_fwd_kernel<DP>, dim3(grid), dim3(256), smem, stream, p));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <int DP>
static int launch_bwd(const AttnParams& p, cudaStream_t stream) {
  constexpr int LDS = DP + 8;
  {
    const long long total = static_cast<long long>(p.B) * p.Sq * p.H;
    CUDA_TRY(launch_pdl(attn_delta_kernel, dim3(static_cast<int>((total + 127) / 128)), dim3(128), 0, stream, p));
  }
  const size_t smem1 = static_cast<size_t>(6 * 64) * LDS * sizeof(bf16) + 4 * 64 * sizeof(float);
  const size_t smem2 = static_cast<size_t>(6 * 64) * LDS * sizeof(bf16);
  static bool set = false;
  if (!set) {
    CUDA_TRY(cudaFuncSetAttribute(attn_bwd_dkdv_kernel<DP>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem1)));
    CUDA_TRY(cudaFuncSetAttribute(attn_bwd_dq_kernel<DP>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem2)));
    set = true;
  }
  CUDA_TRY(launch_pdl(attn_bwd_dkdv_kernel<DP>, dim3(dim3((p.Skv + 63) / 64, p.H, p.B)), dim3(128), smem1, stream, p));
  CUDA_TRY(launch_pdl(attn_bwd_dq_kernel<DP>, dim3(dim3((p.Sq + 63) / 64, p.H, p.B)), dim3(128), smem2, stream, p));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace pcm

namespace pcm {
int attn_fwd_wg(const void* q, const void* k, const void* v, void* out, float* lse, int B, int H, int Sq,
                int Skv, int D, long long ldq, long long ldk, long long ldv, long long ldo, float scale,
                cudaStream_t stream);  // attn_wg.cu
int attn_bwd_wg(const void* q, const void* k, const void* v, const void* dout, const float* lse,
                const float* delta, void* dq, void* dk, void* dv, int B, int H, int Sq, int Skv, int D,
                long long ldq, long long ldk, long long ldv, long long ldo, float scale, cudaStream_t stream);
}
using namespace pcm;

#define DISPATCH_DP(D, CALL)                                                     \
  do {                                                                           \
    if ((D) % 8 != 0) return set_error("attention: head dim must be a multiple of 8"); \
    const int dp_ = ((D) + 15) / 16 * 16;                                        \
    switch (dp_) {                                                               \
      case 16: return CALL<16>(p, st);                                           \
      case 32: return CALL<32>(p, st);                                           \
      case 48: return CALL<48>(p, st);                                           \
      case 64: return CALL<64>(p, st);                                           \
      case 80: return CALL<80>(p, st);                                           \
      case 96: return CALL<96>(p, st);                                           \
      case 128: return CALL<128>(p, st);                                         \
      case 160: return CALL<160>(p, st);                                         \
      default: return set_error("attention: unsupported head dim");              \
    }                                                                            \
  } while (0)

extern "C" int pcm_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse,
                            int B, int H, int Sq, int Skv, int D, int64_t ldq, int64_t ldk,
                            int64_t ldv, int64_t ldo, float scale, void* stream) {
  AttnParams p{};
  p.q = reinterpret_cast<const bf16*>(q);
  p.k = reinterpret_cast<const bf16*>(k);
  p.v = reinterpret_cast<const bf16*>(v);
  p.out = reinterpret_cast<bf16*>(out);
  p.lse = lse;
  p.B = B; p.H = H; p.Sq = Sq; p.Skv = Skv; p.D = D;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.scale = scale;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // wgmma / TMA kernel (d <= 128); returns 1 when the shape or layout is not covered
  const int rc = attn_fwd_wg(q, k, v, out, lse, B, H, Sq, Skv, D, ldq, ldk, ldv, ldo, scale, st);
  if (rc <= 0) return rc;
  DISPATCH_DP(D, launch_fwd);
}

extern "C" int pcm_attn_bwd(const void* q, const void* k, const void* v, const void* o,
                            const void* dout, const float* lse, float* delta, void* dq, void* dk,
                            void* dv, int B, int H, int Sq, int Skv, int D, int64_t ldq,
                            int64_t ldk, int64_t ldv, int64_t ldo, float scale, void* stream) {
  AttnParams p{};
  p.q = reinterpret_cast<const bf16*>(q);
  p.k = reinterpret_cast<const bf16*>(k);
  p.v = reinterpret_cast<const bf16*>(v);
  p.o = reinterpret_cast<const bf16*>(o);
  p.dout = reinterpret_cast<const bf16*>(dout);
  p.lse = const_cast<float*>(lse);
  p.delta = delta;
  p.dq = reinterpret_cast<bf16*>(dq);
  p.dk = reinterpret_cast<bf16*>(dk);
  p.dv = reinterpret_cast<bf16*>(dv);
  p.B = B; p.H = H; p.Sq = Sq; p.Skv = Skv; p.D = D;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.scale = scale;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (D <= 64 && D % 8 == 0) {
    // wgmma / TMA kernels (d <= 64) after delta = rowsum(dO o O); return 1 when the layout is not covered
    const long long total = static_cast<long long>(B) * Sq * H;
    CUDA_TRY(launch_pdl(attn_delta_kernel, dim3(static_cast<unsigned>((total + 127) / 128)), dim3(128), 0, st, p));
    const int rc = attn_bwd_wg(q, k, v, dout, lse, delta, dq, dk, dv, B, H, Sq, Skv, D, ldq, ldk, ldv, ldo, scale, st);
    if (rc <= 0) return rc;
  }
  DISPATCH_DP(D, launch_bwd);
}
