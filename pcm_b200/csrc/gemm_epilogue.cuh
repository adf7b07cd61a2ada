// Epilogue of one 64 x BN accumulator half-tile held in the registers of one consumer warpgroup.
// Two phases per 32-column chunk so that global traffic is coalesced:
//   1. every thread writes its wgmma fragments of the chunk (2 rows x 8 columns) into an fp32 staging
//      tile in shared memory (16-byte chunks XOR-swizzled by row to stay conflict free);
//   2. the 128 threads of the warpgroup re-map to (row, 8-column group): 4 neighbouring lanes cover
//      64 contiguous output bytes of one row, add bias / row vector / residual, apply the activation,
//      store 16 bytes.
//
// The common case - bf16 output, full 32-column chunk, no activation, no split-K - is a compact
// straight-line path and everything else (ragged N, fp32 output, split-K partial sums) lives in one
// out-of-line routine with rolled loops.
#pragma once
#include "gemm_params.h"

namespace pcm {

// Generic phase 2 of one chunk for the calling thread's 2 rows: ragged N, fp32 output, split-K.
// m0: first output row of this warpgroup's half-tile.
static __device__ __noinline__ void gemm_epilogue_rows_generic(const GemmParams& p, const float* sb, int m0,
                                                               int n, int r0, int cg, float* ws) {
#pragma unroll 1
  for (int i = 0; i < 2; ++i) {
    const int rr = r0 + 32 * i;
    const int m = m0 + rr;
    if (m >= p.M) continue;
    const float* srow = sb + rr * 32;
    if (ws) {  // split-K partial sums: plain stores into this split's slice of the workspace (the
               // finalize kernel adds the slices in split order and applies the epilogue)
      const float4 a0 = *reinterpret_cast<const float4*>(srow + ((2 * cg) ^ (rr & 7)) * 4);
      const float4 a1 = *reinterpret_cast<const float4*>(srow + ((2 * cg + 1) ^ (rr & 7)) * 4);
      const float f[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float* wp = ws + static_cast<long long>(m) * p.N + n;
      if (n + 8 <= p.N && (p.N & 3) == 0) {   // two 16-byte stores (rows are 16-byte aligned)
        *reinterpret_cast<float4*>(wp) = make_float4(f[0] * p.alpha, f[1] * p.alpha, f[2] * p.alpha, f[3] * p.alpha);
        *reinterpret_cast<float4*>(wp + 4) = make_float4(f[4] * p.alpha, f[5] * p.alpha, f[6] * p.alpha, f[7] * p.alpha);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (n + e < p.N) wp[e] = f[e] * p.alpha;
      }
      continue;
    }
    const int b = m / p.epiHW;
    const int r = m - b * p.epiHW;
    const int h = r / p.epiW;
    const int w = r - h * p.epiW;
    const long long o = b * p.osB + h * p.osH + w * p.osW;
#pragma unroll 1
    for (int e = 0; e < 8 && n + e < p.N; ++e) {
      float x = srow[((2 * cg + (e >> 2)) ^ (rr & 7)) * 4 + (e & 3)] * p.alpha;
      if (p.bias) x += p.bias[n + e];
      if (p.rowvec) x += __bfloat162float(p.rowvec[b * p.rowvec_ld + n + e]);
      if (p.residual) x += __bfloat162float(p.residual[o + n + e]);
      if (p.act == 1) x = silu_f(x);
      if (p.out_fp32) {
        if (p.round_bf16) x = __bfloat162float(__float2bfloat16_rn(x));
        reinterpret_cast<float*>(p.out)[o + n + e] = x;
      } else {
        reinterpret_cast<bf16*>(p.out)[o + n + e] = __float2bfloat16_rn(x);
      }
    }
  }
}

__device__ __forceinline__ void add_bf16x8(float (&f)[8], const uint4& u) {
  float2 t;
  t = unpack_bf16x2(u.x); f[0] += t.x; f[1] += t.y;
  t = unpack_bf16x2(u.y); f[2] += t.x; f[3] += t.y;
  t = unpack_bf16x2(u.z); f[4] += t.x; f[5] += t.y;
  t = unpack_bf16x2(u.w); f[6] += t.x; f[7] += t.y;
}

// acc: the m64 x BN wgmma accumulator of this warpgroup (rows m0 .. m0 + 63, columns n0 ..);
// sb: the warpgroup's 64 x 32 fp32 staging tile; et: thread index inside the warpgroup;
// bar: named barrier id of the warpgroup.
template <int BN>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmParams& p, int m0, int n0, const float (&acc)[BN / 2],
                                                   float* sb, int et, int bar, float* ws) {
  const bool has_bias = p.bias != nullptr, has_rv = p.rowvec != nullptr;
  // split-K, fp32 output and the SiLU epilogue (time-embedding MLP, M = batch) take the generic path
  const bool fast_ok = p.ws == nullptr && !p.out_fp32 && p.act == 0;
  const bool has_res = p.residual != nullptr && fast_ok;
  const int cg = et & 3;   // phase 2: 8-column group inside the 32-column chunk
  const int r0 = et >> 2;  // phase 2: rows r0 and r0 + 32
  long long off[2];
  const bf16* rvp[2];
  bool valid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + r0 + 32 * i;
    valid[i] = m < p.M;
    off[i] = 0;
    rvp[i] = nullptr;
    if (valid[i]) {
      const int b = m / p.epiHW;
      const int r = m - b * p.epiHW;
      const int h = r / p.epiW;
      const int w = r - h * p.epiW;
      off[i] = b * p.osB + h * p.osH + w * p.osW;
      if (has_rv) rvp[i] = p.rowvec + b * p.rowvec_ld;
    }
  }
  constexpr int kChunks = BN / 32;
  const uint32_t sb_u32 = smem_u32(sb);
  // phase 1: fragment rows (et / 32) * 16 + (et % 32) / 4 (+8), columns 8 q + 2 (et % 4) (+1)
  const int frow = ((et >> 5) << 4) + ((et & 31) >> 2);
  const uint32_t st0 = sb_u32 + frow * 128, st1 = st0 + 8 * 128;
  const uint32_t st_x = (frow & 7) << 4;                 // rows frow and frow + 8 share (row & 7)
  const uint32_t st_in = (et & 1) << 3;                  // byte offset inside the 16-byte chunk
  const int st_c = (et & 3) >> 1;                        // 16-byte chunk of the column pair inside 8 columns
  const uint32_t ld_a0 = sb_u32 + r0 * 128 + (((2 * cg) ^ (r0 & 7)) << 4);   // phase 2
  const uint32_t ld_a1 = sb_u32 + r0 * 128 + (((2 * cg + 1) ^ (r0 & 7)) << 4);
  // Residual reads come from HBM: the reads of TWO chunks are kept in flight.  (out may alias
  // residual for in-place accumulation: every element is read and later written by the same
  // thread, tiles are disjoint.)
  uint4 rcur[2], rnext[2];
  auto load_res = [&](uint4 (&dst)[2], int j) {
    const int n = n0 + j * 32 + cg * 8;
    if (j < kChunks && n + 8 <= p.N) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (valid[i]) dst[i] = *reinterpret_cast<const uint4*>(p.residual + off[i] + n);
    }
  };
  if (has_res) {
    load_res(rcur, 0);
    load_res(rnext, 1);
  }
#pragma unroll 1
  for (int j = 0; j < kChunks; ++j) {
    const int n = n0 + j * 32 + cg * 8;
    const bool fast = fast_ok && (n0 + j * 32 + 32 <= p.N);  // uniform over the warpgroup
    // bias / row vectors are L2 resident: issued per chunk, ahead of the staging writes
    float4 bia0 = make_float4(0.f, 0.f, 0.f, 0.f), bia1 = bia0;
    uint4 rrv[2];
    if (fast) {
      if (has_bias) {
        bia0 = *reinterpret_cast<const float4*>(p.bias + n);
        bia1 = *reinterpret_cast<const float4*>(p.bias + n + 4);
      }
      if (has_rv) {
#pragma unroll
        for (int i = 0; i < 2; ++i)
          if (valid[i]) rrv[i] = *reinterpret_cast<const uint4*>(rvp[i] + n);
      }
    }
    // phase 1 (registers are indexed at compile time: the chunk is selected by predicate)
#pragma unroll
    for (int jj = 0; jj < kChunks; ++jj) {
      if (jj != j) continue;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t c = (static_cast<uint32_t>(2 * q + st_c) << 4) ^ st_x;
        const float* a = &acc[16 * jj + 4 * q];
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(st0 + c + st_in), "f"(a[0]), "f"(a[1]) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(st1 + c + st_in), "f"(a[2]), "f"(a[3]) : "memory");
      }
    }
    asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");  // staging tile written
    if (fast) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;
        // rows r0 and r0 + 32 share (row & 7): same swizzle, 4 KB apart
        const float4 a0 = lds128(ld_a0 + i * 4096);
        const float4 a1 = lds128(ld_a1 + i * 4096);
        float f[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        if (p.alpha != 1.0f) {
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] *= p.alpha;
        }
        f[0] += bia0.x; f[1] += bia0.y; f[2] += bia0.z; f[3] += bia0.w;
        f[4] += bia1.x; f[5] += bia1.y; f[6] += bia1.z; f[7] += bia1.w;
        if (has_rv) add_bf16x8(f, rrv[i]);
        if (has_res) add_bf16x8(f, rcur[i]);
        uint4 u;
        u.x = pack_bf16x2(f[0], f[1]);
        u.y = pack_bf16x2(f[2], f[3]);
        u.z = pack_bf16x2(f[4], f[5]);
        u.w = pack_bf16x2(f[6], f[7]);
        *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(p.out) + off[i] + n) = u;
      }
      if (has_res) {
#pragma unroll
        for (int i = 0; i < 2; ++i) rcur[i] = rnext[i];
        load_res(rnext, j + 2);
      }
    } else if (n < p.N) {
      gemm_epilogue_rows_generic(p, sb, m0, n, r0, cg, ws);
    }
    // staging tile consumed: the warpgroup may overwrite it in its next chunk
    asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
  }
}

}  // namespace pcm
