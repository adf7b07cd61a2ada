// GroupNorm(+SiLU) and LayerNorm, forward and input-gradient, on NHWC bf16 activations.
// HBM-bound kernels: 16-byte vector loads along the contiguous channel dimension, fp32 statistics,
// warp/shared-memory reductions, one bf16 rounding at the output.
//
// Replaces the ATen group_norm / layer_norm / silu launches inside diffusers' ResnetBlock2D,
// Transformer2DModel and BasicTransformerBlock (called from train_pcm_lora_sd15.py:1192-1198,
// 1219-1244, 1263-1268) and their autograd backward (:1296).  GroupNorm reads an optional second
// source so the up-block skip concat torch.cat([h, res], dim=1) is never materialised twice.
#include "common.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"

namespace pcm {

// ------------------------------------------------------------------------------------------
// GroupNorm statistics: stats[b, g] = (mean, rstd) over HW x (C/G) elements.
//
// Reproducible and cancellation free (torch / diffusers use a Welford-style computation):
//   * every block accumulates, per channel, sums of (x - pivot) and (x - pivot)^2 with the pivot =
//     the channel's value at the first pixel of the image, so |x - pivot| = O(sigma) even when
//     |mean| >> sigma; the channels of a group are merged with Chan's parallel-variance formula;
//   * the block writes its (mean, M2) per group to a workspace slot (no atomics on data); the LAST
//     block of an image to finish (a self-resetting counter) merges the per-block partials in block
//     order, so the result does not depend on the order in which blocks ran.
// ------------------------------------------------------------------------------------------
constexpr int kGnMaxC = 2560;
constexpr int kGnStage = 4096;   // ny * C <= 4096 floats of per-thread partials (see gn_launch_cfg)
constexpr int kGnMaxB = 1024;    // counters per kernel family in the workspace

__device__ __forceinline__ const bf16* gn_src(const bf16* x1, const bf16* x2, int C1, int C2,
                                              long long pix, int c) {
  return c < C1 ? x1 + pix * C1 + c : x2 + pix * C2 + (c - C1);
}

// true for exactly one block per image: the last one to arrive; makes the other blocks' global
// writes visible to it
__device__ __forceinline__ bool gn_last_block(unsigned* counter, unsigned nblk) {
  __shared__ unsigned s_old;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_old = atomicAdd(counter, 1u);
  __syncthreads();
  const bool last = s_old == nblk - 1;
  if (last) __threadfence();
  return last;
}

// Chan et al. pairwise update of (count, mean, M2) with a second partial (nb may be 0)
__device__ __forceinline__ void chan_merge(float& na, float& mean, float& m2, float nb, float mb,
                                           float m2b) {
  const float nn = na + nb;
  if (nn <= 0.f) return;
  const float d = mb - mean;
  const float f = nb / nn;
  mean += d * f;
  m2 += m2b + d * d * na * f;
  na = nn;
}

__global__ void __launch_bounds__(512, 2) gn_stats_kernel(const bf16* __restrict__ x1, const bf16* __restrict__ x2, int C1,
                                int C2, int HW, int G, int pix_per_block, float eps,
                                float* __restrict__ part, unsigned* __restrict__ counters,
                                float* __restrict__ stats) {
  griddep_sync();
  // per-thread partials are staged as [ty][channel] (plain stores) and summed in a fixed order
  __shared__ float s_sum[kGnStage];
  __shared__ float s_sq[kGnStage];
  __shared__ float s_piv[kGnMaxC];
  const int C = C1 + C2;
  const int b = blockIdx.y;
  const int nblk = gridDim.x;
  const int nvec = C >> 3;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const int ny = blockDim.x / nvec;
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  float a[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = q[i] = 0.f;
  if (ty < ny) {
    const int c = tx * 8;
    float piv[8];
    {
      const uint4 u = *reinterpret_cast<const uint4*>(
          gn_src(x1, x2, C1, C2, static_cast<long long>(b) * HW, c));
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(w[i]);
        piv[2 * i] = f.x;
        piv[2 * i + 1] = f.y;
      }
    }
    // four independent 16-byte loads in flight per thread
    for (int p = p0 + ty; p < p1; p += 4 * ny) {
      uint4 u[4];
      bool ok[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int pp = p + k * ny;
        ok[k] = pp < p1;
        u[k] = make_uint4(0, 0, 0, 0);
        if (ok[k])
          u[k] = *reinterpret_cast<const uint4*>(
              gn_src(x1, x2, C1, C2, static_cast<long long>(b) * HW + pp, c));
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!ok[k]) continue;
        const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16x2(w[i]);
          const float d0 = f.x - piv[2 * i], d1 = f.y - piv[2 * i + 1];
          a[2 * i] += d0; q[2 * i] += d0 * d0;
          a[2 * i + 1] += d1; q[2 * i + 1] += d1 * d1;
        }
      }
    }
    *reinterpret_cast<float4*>(&s_sum[ty * C + c]) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(&s_sum[ty * C + c + 4]) = make_float4(a[4], a[5], a[6], a[7]);
    *reinterpret_cast<float4*>(&s_sq[ty * C + c]) = make_float4(q[0], q[1], q[2], q[3]);
    *reinterpret_cast<float4*>(&s_sq[ty * C + c + 4]) = make_float4(q[4], q[5], q[6], q[7]);
    if (ty == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) s_piv[c + i] = piv[i];
    }
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int y = 0; y < ny; ++y) {
      s += s_sum[y * C + ch];
      ss += s_sq[y * C + ch];
    }
    s_sum[ch] = s;   // row 0 now holds the block totals (each thread only touches its own column)
    s_sq[ch] = ss;
  }
  __syncthreads();
  const int cpg = C / G;
  const float n = static_cast<float>(p1 - p0);   // pixels per channel in this block
  const float inv_n = 1.f / n;
  // per channel: (mean, M2) from the pivot-shifted sums, all threads (no divisions in the loops)
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    const float s = s_sum[ch];
    const float m2 = s_sq[ch] - s * s * inv_n;
    s_sum[ch] = s_piv[ch] + s * inv_n;
    s_sq[ch] = m2;
  }
  __syncthreads();
  // per group: Chan merge of its channels (equal counts)
  const float inv_cpg = 1.f / static_cast<float>(cpg);
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float msum = 0.f, m2 = 0.f;
    for (int i = 0; i < cpg; ++i) {
      msum += s_sum[g * cpg + i];
      m2 += s_sq[g * cpg + i];
    }
    const float mg = msum * inv_cpg;
    float dev = 0.f;
    for (int i = 0; i < cpg; ++i) {
      const float d = s_sum[g * cpg + i] - mg;
      dev += d * d;
    }
    float* o = part + (static_cast<long long>(b * nblk + blockIdx.x) * G + g) * 2;
    o[0] = mg;
    o[1] = m2 + n * dev;
  }
  if (!gn_last_block(&counters[b], nblk)) return;
  // merge the per-block partials: staged in shared memory by all threads (one round of loads),
  // then 8 lanes per group fold blocks lane, lane + 8, ... in order and combine in a fixed
  // shuffle tree - the result is independent of the order in which the blocks ran
  for (int i = threadIdx.x; i < nblk * G; i += blockDim.x) {
    const float* o = part + (static_cast<long long>(b) * nblk * G + i) * 2;
    s_sum[i] = __ldcg(o);
    s_sq[i] = __ldcg(o + 1);
  }
  __syncthreads();
  if (threadIdx.x < G * 8) {   // whole warps (G * 8 is a multiple of 32 for G = 4 k)
    const int g = threadIdx.x >> 3, j = threadIdx.x & 7;
    float na = 0.f, mean = 0.f, m2 = 0.f;
    for (int k = j; k < nblk; k += 8)
      chan_merge(na, mean, m2,
                 static_cast<float>(min(HW, (k + 1) * pix_per_block) - k * pix_per_block) * cpg,
                 s_sum[k * G + g], s_sq[k * G + g]);
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const float nb = __shfl_xor_sync(0xffffffffu, na, o);
      const float mb = __shfl_xor_sync(0xffffffffu, mean, o);
      const float m2b = __shfl_xor_sync(0xffffffffu, m2, o);
      // both partners compute the same merge (lower lane's partial first): symmetric result
      if (j & o) {
        float ta = nb, tm = mb, t2 = m2b;
        chan_merge(ta, tm, t2, na, mean, m2);
        na = ta; mean = tm; m2 = t2;
      } else {
        chan_merge(na, mean, m2, nb, mb, m2b);
      }
    }
    if (j == 0) {
      stats[(b * G + g) * 2] = mean;
      stats[(b * G + g) * 2 + 1] = rsqrtf(fmaxf(m2 / na, 0.f) + eps);
    }
  }
  if (threadIdx.x == 0) counters[b] = 0;   // ready for the next launch
}

// out = [silu]( (x - mean) * rstd * gamma + beta ), bf16.  Same thread -> channel-vector mapping as
// gn_stats_kernel: each thread folds the statistics of its 8 channels into (scale, shift) once and
// then streams pixels (16-byte load, 8 FMAs, 16-byte store), four pixels in flight.
__global__ void gn_apply_kernel(const bf16* __restrict__ x1, const bf16* __restrict__ x2, int C1,
                                int C2, int HW, int G, int pix_per_block,
                                const float* __restrict__ stats, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int silu,
                                bf16* __restrict__ out) {
  griddep_sync();
  const int C = C1 + C2;
  const int b = blockIdx.y;
  const int nvec = C >> 3;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const int ny = blockDim.x / nvec;
  const int cpg = C / G;
  const int c = tx * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c + i) / cpg;
    const float mean = stats[(b * G + g) * 2];
    const float rstd = stats[(b * G + g) * 2 + 1];
    sc[i] = rstd * gamma[c + i];
    sh[i] = beta[c + i] - mean * sc[i];
  }
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  constexpr int U = 4;  // independent 16-byte loads in flight per thread
  for (int p = p0 + ty; p < p1; p += U * ny) {
    uint4 u[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int pp = p + k * ny;
      if (pp < p1)
        u[k] = *reinterpret_cast<const uint4*>(gn_src(x1, x2, C1, C2, static_cast<long long>(b) * HW + pp, c));
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int pp = p + k * ny;
      if (pp >= p1) break;
      const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
      float f[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 t = unpack_bf16x2(w[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float y = f[i] * sc[i] + sh[i];
        if (silu) y = silu_f(y);
        f[i] = y;
      }
      uint4 o;
      o.x = pack_bf16x2(f[0], f[1]);
      o.y = pack_bf16x2(f[2], f[3]);
      o.z = pack_bf16x2(f[4], f[5]);
      o.w = pack_bf16x2(f[6], f[7]);
      *reinterpret_cast<uint4*>(out + (static_cast<long long>(b) * HW + pp) * C + c) = o;
    }
  }
}

// backward reductions: red[b, g] = (sum gamma*dyh, sum gamma*dyh*xhat), dyh = dy * silu'(pre);
// per-block partials merged in block order by the last block of the image (see gn_stats_kernel)
__global__ void __launch_bounds__(512, 2) gn_bwd_stats_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x1,
                                    const bf16* __restrict__ x2, int C1, int C2, int HW, int G,
                                    int pix_per_block, const float* __restrict__ stats,
                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                    int silu, float* __restrict__ part,
                                    unsigned* __restrict__ counters, float* __restrict__ red) {
  griddep_sync();
  __shared__ float s_a[kGnStage];
  __shared__ float s_b[kGnStage];
  const int C = C1 + C2;
  const int b = blockIdx.y;
  const int nblk = gridDim.x;
  const int nvec = C >> 3;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const int ny = blockDim.x / nvec;
  const int cpg = C / G;
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  if (ty < ny) {
    const int c = tx * 8;
    // folded per-channel constants: pre = xhat*gamma + beta = x*U + V.  The second reduction is
    // accumulated as sum(g * pre) (pre is O(1), no cancellation) and converted at the end:
    // sum(g * xhat) = (sum(g * pre) - beta * sum(g)) / gamma.   g = dy * silu'(pre) * gamma
    float U[8], V[8], gm[8], a[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int g = (c + i) / cpg;
      const float mean = stats[(b * G + g) * 2];
      const float rstd = stats[(b * G + g) * 2 + 1];
      gm[i] = gamma[c + i];
      U[i] = rstd * gm[i];
      V[i] = beta[c + i] - mean * U[i];
      a[i] = q[i] = 0.f;
    }
    for (int p = p0 + ty; p < p1; p += ny) {
      const long long pix = static_cast<long long>(b) * HW + p;
      const uint4 u = *reinterpret_cast<const uint4*>(gn_src(x1, x2, C1, C2, pix, c));
      const uint4 d = *reinterpret_cast<const uint4*>(dy + pix * C + c);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      const uint32_t dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 xf = unpack_bf16x2(w[i]);
        const float2 df = unpack_bf16x2(dw[i]);
        const float xs[2] = {xf.x, xf.y}, ds[2] = {df.x, df.y};
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int k = 2 * i + j;
          const float pre = fmaf(xs[j], U[k], V[k]);
          float g = ds[j] * gm[k];
          if (silu) g *= dsilu_f(pre);
          a[k] += g;
          q[k] = fmaf(g, pre, q[k]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)   // sum(g * pre) -> sum(g * xhat)
      q[i] = gm[i] != 0.f ? (q[i] - beta[c + i] * a[i]) / gm[i] : 0.f;
    *reinterpret_cast<float4*>(&s_a[ty * C + c]) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(&s_a[ty * C + c + 4]) = make_float4(a[4], a[5], a[6], a[7]);
    *reinterpret_cast<float4*>(&s_b[ty * C + c]) = make_float4(q[0], q[1], q[2], q[3]);
    *reinterpret_cast<float4*>(&s_b[ty * C + c + 4]) = make_float4(q[4], q[5], q[6], q[7]);
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int y = 0; y < ny; ++y) {
      s += s_a[y * C + ch];
      ss += s_b[y * C + ch];
    }
    s_a[ch] = s;
    s_b[ch] = ss;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int i = 0; i < cpg; ++i) {
      s += s_a[g * cpg + i];
      ss += s_b[g * cpg + i];
    }
    float* o = part + (static_cast<long long>(b * nblk + blockIdx.x) * G + g) * 2;
    o[0] = s;
    o[1] = ss;
  }
  if (!gn_last_block(&counters[b], nblk)) return;
  __syncthreads();
  for (int i = threadIdx.x; i < nblk * G; i += blockDim.x) {
    const float* o = part + (static_cast<long long>(b) * nblk * G + i) * 2;
    s_a[i] = __ldcg(o);
    s_b[i] = __ldcg(o + 1);
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int k = 0; k < nblk; ++k) {   // block order: independent of the execution order
      s += s_a[k * G + g];
      ss += s_b[k * G + g];
    }
    red[(b * G + g) * 2] = s;
    red[(b * G + g) * 2 + 1] = ss;
  }
  if (threadIdx.x == 0) counters[b] = 0;
}

// dx = rstd * (gamma*dyh - (s1 + xhat*s2)/n) (+ add); written to dx1 (first C1 channels) and
// dx2 (remaining C2 channels).  Per-thread channel constants hoisted like gn_apply_kernel.
// colsum (optional): per-image column sums of dx, again as per-block partials merged in block
// order by the last block of the image.
__global__ void __launch_bounds__(512, 2) gn_bwd_apply_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x1,
                                    const bf16* __restrict__ x2, int C1, int C2, int HW, int G,
                                    int pix_per_block, const float* __restrict__ stats,
                                    const float* __restrict__ red, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, int silu,
                                    const bf16* __restrict__ add, bf16* __restrict__ dx1,
                                    bf16* __restrict__ dx2, float* __restrict__ colsum,
                                    float* __restrict__ cpart, unsigned* __restrict__ counters) {
  griddep_sync();
  __shared__ float s_cs[kGnStage];
  const int C = C1 + C2;
  const int b = blockIdx.y;
  const int nblk = gridDim.x;
  const int nvec = C >> 3;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const int ny = blockDim.x / nvec;
  const int cpg = C / G;
  const float inv_n = 1.f / (static_cast<float>(HW) * cpg);
  const int c = tx * 8;
  float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  // folded per-channel constants (4 instead of 6 registers per channel):
  //   pre = x*U + V (pre-activation), dx = dy * silu'(pre) * U + x*P + Q (+ add)
  //   U = rstd*gamma, V = beta - mean*U, P = -rstd^2 * s2, Q = -rstd*s1 - mean*P
  float U[8], V[8], P[8], Q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c + i) / cpg;
    const float mean = stats[(b * G + g) * 2];
    const float rstd = stats[(b * G + g) * 2 + 1];
    const float s1 = red[(b * G + g) * 2] * inv_n;
    const float s2 = red[(b * G + g) * 2 + 1] * inv_n;
    U[i] = rstd * gamma[c + i];
    V[i] = beta[c + i] - mean * U[i];
    P[i] = -rstd * rstd * s2;
    Q[i] = -rstd * s1 - mean * P[i];
  }
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  for (int p = p0 + ty; p < p1; p += ny) {
    const long long pix = static_cast<long long>(b) * HW + p;
    const uint4 u = *reinterpret_cast<const uint4*>(gn_src(x1, x2, C1, C2, pix, c));
    const uint4 d = *reinterpret_cast<const uint4*>(dy + pix * C + c);
    uint4 ad = make_uint4(0, 0, 0, 0);
    if (add) ad = *reinterpret_cast<const uint4*>(add + pix * C + c);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    const uint32_t dw[4] = {d.x, d.y, d.z, d.w};
    const uint32_t aw[4] = {ad.x, ad.y, ad.z, ad.w};
    float o[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 xf = unpack_bf16x2(w[i]);
      const float2 df = unpack_bf16x2(dw[i]);
      const float2 af = unpack_bf16x2(aw[i]);
      const float xs[2] = {xf.x, xf.y}, ds[2] = {df.x, df.y}, as[2] = {af.x, af.y};
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int k = 2 * i + j;
        float gg = ds[j] * U[k];
        if (silu) gg *= dsilu_f(fmaf(xs[j], U[k], V[k]));
        o[k] = gg + fmaf(xs[j], P[k], Q[k]) + as[j];
      }
    }
    uint4 ov;
    ov.x = pack_bf16x2(o[0], o[1]);
    ov.y = pack_bf16x2(o[2], o[3]);
    ov.z = pack_bf16x2(o[4], o[5]);
    ov.w = pack_bf16x2(o[6], o[7]);
    if (c < C1)
      *reinterpret_cast<uint4*>(dx1 + pix * C1 + c) = ov;
    else
      *reinterpret_cast<uint4*>(dx2 + pix * C2 + (c - C1)) = ov;
    if (colsum) {
#pragma unroll
      for (int k = 0; k < 8; ++k) cs[k] += o[k];
    }
  }
  if (!colsum) return;   // uniform over the grid
  // per-image column sums of dx (time-embedding gradient), fp32, fixed summation order
  if (ty < ny) {
    *reinterpret_cast<float4*>(&s_cs[ty * C + c]) = make_float4(cs[0], cs[1], cs[2], cs[3]);
    *reinterpret_cast<float4*>(&s_cs[ty * C + c + 4]) = make_float4(cs[4], cs[5], cs[6], cs[7]);
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    float s = 0.f;
    for (int y = 0; y < ny; ++y) s += s_cs[y * C + ch];
    cpart[static_cast<long long>(b * nblk + blockIdx.x) * C + ch] = s;
  }
  if (!gn_last_block(&counters[b], nblk)) return;
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    float s = 0.f;
#pragma unroll 8
    for (int k = 0; k < nblk; ++k) s += __ldcg(cpart + static_cast<long long>(b * nblk + k) * C + ch);
    colsum[b * C + ch] = s;
  }
  if (threadIdx.x == 0) counters[b] = 0;
}

// ------------------------------------------------------------------------------------------
// LayerNorm over the channel dimension.  LPR lanes cooperate on one token row (C/8 <= 5 * LPR
// 16-byte vectors, 5 independent loads per lane), 32 / LPR rows per warp; group reductions by
// xor-shuffles below LPR.  SD1.5: C = 320 / 640 / 1280 -> LPR = 8 / 16 / 32, perfectly balanced.
// ------------------------------------------------------------------------------------------
constexpr int kLnMaxVec = 5;

template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int LPR>
__global__ void __launch_bounds__(256, 4) ln_fwd_kernel(const bf16* __restrict__ x, int M, int C,
                              const float* __restrict__ gamma, const float* __restrict__ beta,
                              float eps, bf16* __restrict__ out, float* __restrict__ stats) {
  griddep_sync();
  constexpr int RPW = 32 / LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR;
  const int nvec = C >> 3;
  // grid-stride over groups of RPW rows: a few fat blocks per SM instead of thousands of one-shot blocks
  for (int warp = warp0; warp * RPW < M; warp += nwarps) {
  const int r = warp * RPW + lane / LPR;
  const bool rvalid = r < M;
  const bf16* row = x + static_cast<long long>(rvalid ? r : 0) * C;
  float f[kLnMaxVec][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = sub + i * LPR;
    if (v < nvec) {
      const uint4 u = *reinterpret_cast<const uint4*>(row + v * 8);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = unpack_bf16x2(w[j]);
        f[i][2 * j] = t.x;
        f[i][2 * j + 1] = t.y;
        s += t.x + t.y;
      }
    }
  }
  const float mean = group_sum<LPR>(s) / C;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = sub + i * LPR;
    if (v < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[i][j] - mean;
        ss += d * d;
      }
    }
  }
  const float rstd = rsqrtf(group_sum<LPR>(ss) / C + eps);
  if (!rvalid) continue;
  if (sub == 0 && stats) {
    stats[r * 2] = mean;
    stats[r * 2 + 1] = rstd;
  }
  bf16* orow = out + static_cast<long long>(r) * C;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = sub + i * LPR;
    if (v < nvec) {
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + v * 8);
      const float4 g1 = *reinterpret_cast<const float4*>(gamma + v * 8 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(beta + v * 8);
      const float4 b1 = *reinterpret_cast<const float4*>(beta + v * 8 + 4);
      const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bt[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (f[i][j] - mean) * rstd * gm[j] + bt[j];
      uint4 u;
      u.x = pack_bf16x2(o[0], o[1]);
      u.y = pack_bf16x2(o[2], o[3]);
      u.z = pack_bf16x2(o[4], o[5]);
      u.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(orow + v * 8) = u;
    }
  }
  }
}

// dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)) (+ add)
template <int LPR>
__global__ void ln_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, int M, int C,
                              const float* __restrict__ gamma, const float* __restrict__ stats,
                              const bf16* __restrict__ add, bf16* __restrict__ dx) {
  griddep_sync();
  constexpr int RPW = 32 / LPR;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR;
  const int r = warp * RPW + lane / LPR;
  const bool rvalid = r < M;
  const int nvec = C >> 3;
  const long long base = static_cast<long long>(rvalid ? r : 0) * C;
  const float mean = stats[(rvalid ? r : 0) * 2], rstd = stats[(rvalid ? r : 0) * 2 + 1];
  float g[kLnMaxVec][8], xh[kLnMaxVec][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = sub + i * LPR;
    if (v < nvec) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + base + v * 8);
      const uint4 d = *reinterpret_cast<const uint4*>(dy + base + v * 8);
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + v * 8);
      const float4 g1 = *reinterpret_cast<const float4*>(gamma + v * 8 + 4);
      const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      const uint32_t dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 xf = unpack_bf16x2(w[j]);
        const float2 df = unpack_bf16x2(dw[j]);
        xh[i][2 * j] = (xf.x - mean) * rstd;
        xh[i][2 * j + 1] = (xf.y - mean) * rstd;
        g[i][2 * j] = df.x * gm[2 * j];
        g[i][2 * j + 1] = df.y * gm[2 * j + 1];
        s1 += g[i][2 * j] + g[i][2 * j + 1];
        s2 += g[i][2 * j] * xh[i][2 * j] + g[i][2 * j + 1] * xh[i][2 * j + 1];
      }
    }
  }
  s1 = group_sum<LPR>(s1) / C;
  s2 = group_sum<LPR>(s2) / C;
  if (!rvalid) return;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = sub + i * LPR;
    if (v < nvec) {
      float o[8];
      float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (add) {
        const uint4 u = *reinterpret_cast<const uint4*>(add + base + v * 8);
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 t = unpack_bf16x2(w[j]);
          a[2 * j] = t.x;
          a[2 * j + 1] = t.y;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (g[i][j] - s1 - xh[i][j] * s2) + a[j];
      uint4 u;
      u.x = pack_bf16x2(o[0], o[1]);
      u.y = pack_bf16x2(o[2], o[3]);
      u.z = pack_bf16x2(o[4], o[5]);
      u.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(dx + base + v * 8) = u;
    }
  }
}

static inline int ln_lpr(int C) {
  const int nvec = C / 8;
  if (nvec <= 8 * kLnMaxVec) return 8;
  if (nvec <= 16 * kLnMaxVec) return 16;
  return 32;
}

static int gn_launch_cfg(int C, int HW, int B, int* threads, int* ppb, int* nblk) {
  const int nvec = C / 8;
  if (C % 8 != 0 || C > kGnMaxC || nvec > 1024) return set_error("groupnorm: unsupported C");
  int ny = 512 / nvec;      // ny * nvec <= 512 threads  =>  ny * C <= 4096 staged floats
  if (ny < 1) ny = 1;
  *threads = nvec * ny;
  // ONE wave of blocks at two resident blocks per SM (all four kernels are built for <= 64 registers),
  // which also keeps the number of partials to merge small:
  // the total block count is at most 2 x 2 x SMs, so there is no third, nearly empty wave (ncu showed
  // the SMs idle for 36 % of the kernel with 600 blocks on 296 slots)
  int target_blocks = (2 * num_sms()) / B;
  if (target_blocks < 1) target_blocks = 1;
  int p = (HW + target_blocks - 1) / target_blocks;
  if (p < ny * 4) p = ny * 4;
  if ((HW + p - 1) / p > 128) p = (HW + 127) / 128;   // partials are merged through kGnStage floats
  *ppb = p;
  *nblk = (HW + p - 1) / p;
  return 0;
}

}  // namespace pcm

using namespace pcm;

// Workspace layout (caller-owned, zero-initialised ONCE; the kernels leave the counters at zero):
//   uint32 counters[3][kGnMaxB]  (fwd stats, bwd stats, bwd column sums)
//   float  partials[...]         per-block partial statistics / column sums
static inline size_t gn_ws_need(int B, int nblk, int C, int G) {
  return sizeof(unsigned) * 3 * kGnMaxB +
         sizeof(float) * static_cast<size_t>(B) * nblk * (2 * G + C);
}

extern "C" int64_t pcm_groupnorm_ws_bytes(int B, int HW, int C, int G) {
  int threads, ppb, nblk;
  // an upper bound: a launch over B images never uses more blocks per image than a single-image
  // launch would
  if (gn_launch_cfg(C, HW, 1, &threads, &ppb, &nblk)) return -1;
  return static_cast<int64_t>(gn_ws_need(B, nblk, C, G));
}

extern "C" int pcm_groupnorm_fwd(const void* x1_, const void* x2_, int C1, int C2, int B, int HW,
                                 int G, const float* gamma, const float* beta, float eps, int silu,
                                 void* out_, float* stats, void* ws, int64_t ws_bytes,
                                 void* stream_) {
  return pcm_groupnorm_fwd_part(x1_, x2_, C1, C2, B, B, HW, G, gamma, beta, eps, silu, out_, stats, ws,
                                ws_bytes, stream_);
}

extern "C" int pcm_groupnorm_fwd_part(const void* x1_, const void* x2_, int C1, int C2, int B,
                                      int part_B, int HW, int G, const float* gamma, const float* beta,
                                      float eps, int silu, void* out_, float* stats, void* ws,
                                      int64_t ws_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int C = C1 + C2;
  if (C % G != 0 || C1 % 8 != 0 || C2 % 8 != 0) return set_error("groupnorm: bad channel split");
  if (B > kGnMaxB) return set_error("groupnorm: batch too large for the counter workspace");
  if (part_B < B) return set_error("groupnorm: part_B must be >= B");
  const bf16* x1 = reinterpret_cast<const bf16*>(x1_);
  const bf16* x2 = reinterpret_cast<const bf16*>(x2_);
  bf16* out = reinterpret_cast<bf16*>(out_);
  unsigned* counters = reinterpret_cast<unsigned*>(ws);
  float* part = reinterpret_cast<float*>(counters + 3 * kGnMaxB);
  int threads, ppb, nblk;
  // the per-image partition (pixels per block) is the one a launch over part_B images would use
  if (int rc = gn_launch_cfg(C, HW, part_B, &threads, &ppb, &nblk)) return rc;
  if (ws == nullptr || static_cast<size_t>(ws_bytes) < gn_ws_need(B, nblk, C, G))
    return set_error("groupnorm: workspace too small (see pcm_groupnorm_ws_bytes)");
  CUDA_TRY(launch_pdl(gn_stats_kernel, dim3(nblk, B), dim3(threads), 0, stream, x1, x2, C1, C2,
                      HW, G, ppb, eps, part, counters, stats));
  CUDA_TRY(launch_pdl(gn_apply_kernel, dim3(nblk, B), dim3(threads), 0, stream, x1, x2, C1, C2,
                      HW, G, ppb, static_cast<const float*>(stats), gamma, beta, silu, out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_groupnorm_bwd(const void* dy_, const void* x1_, const void* x2_, int C1, int C2,
                                 int B, int HW, int G, const float* gamma, const float* beta,
                                 float eps, int silu, const float* stats, float* red,
                                 const void* add_, void* dx1_, void* dx2_, float* colsum,
                                 void* ws, int64_t ws_bytes, void* stream_) {
  (void)eps;  // folded into stats (mean, rstd) by the forward
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int C = C1 + C2;
  // the same channel split as the forward: each thread's 16-byte vectors must lie in x1 or x2 entirely
  if (C % G != 0 || C1 % 8 != 0 || C2 % 8 != 0) return set_error("groupnorm: bad channel split");
  if (B > kGnMaxB) return set_error("groupnorm: batch too large for the counter workspace");
  const bf16* dy = reinterpret_cast<const bf16*>(dy_);
  const bf16* x1 = reinterpret_cast<const bf16*>(x1_);
  const bf16* x2 = reinterpret_cast<const bf16*>(x2_);
  const bf16* add = reinterpret_cast<const bf16*>(add_);
  bf16* dx1 = reinterpret_cast<bf16*>(dx1_);
  bf16* dx2 = reinterpret_cast<bf16*>(dx2_);
  unsigned* counters = reinterpret_cast<unsigned*>(ws);
  float* part = reinterpret_cast<float*>(counters + 3 * kGnMaxB);
  int threads, ppb, nblk;
  if (int rc = gn_launch_cfg(C, HW, B, &threads, &ppb, &nblk)) return rc;
  if (ws == nullptr || static_cast<size_t>(ws_bytes) < gn_ws_need(B, nblk, C, G))
    return set_error("groupnorm: workspace too small (see pcm_groupnorm_ws_bytes)");
  float* cpart = part + static_cast<size_t>(B) * nblk * 2 * G;
  CUDA_TRY(launch_pdl(gn_bwd_stats_kernel, dim3(nblk, B), dim3(threads), 0, stream, dy, x1, x2, C1, C2,
                      HW, G, ppb, stats, gamma, beta, silu, part, counters + kGnMaxB, red));
  CUDA_TRY(launch_pdl(gn_bwd_apply_kernel, dim3(nblk, B), dim3(threads), 0, stream, dy, x1, x2, C1, C2,
                      HW, G, ppb, stats, static_cast<const float*>(red), gamma, beta, silu, add, dx1, dx2,
                      colsum, cpart, counters + 2 * kGnMaxB));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_layernorm_fwd(const void* x, int M, int C, const float* gamma,
                                 const float* beta, float eps, void* out, float* stats,
                                 void* stream_) {
  if (C % 8 != 0 || C > kLnMaxVec * 256) return set_error("layernorm: unsupported C");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int wpb = 8, lpr = ln_lpr(C);
  const int rows_per_block = wpb * (32 / lpr);
  int grid = (M + rows_per_block - 1) / rows_per_block;
  if (grid > 4 * num_sms()) grid = 4 * num_sms();   // 4 resident blocks per SM, grid-stride
  const bf16* xp = reinterpret_cast<const bf16*>(x);
  bf16* op = reinterpret_cast<bf16*>(out);
  if (lpr == 8) CUDA_TRY(launch_pdl(ln_fwd_kernel<8>, dim3(grid), dim3(wpb * 32), 0, stream, xp, M, C, gamma, beta, eps, op, stats));
  else if (lpr == 16) CUDA_TRY(launch_pdl(ln_fwd_kernel<16>, dim3(grid), dim3(wpb * 32), 0, stream, xp, M, C, gamma, beta, eps, op, stats));
  else CUDA_TRY(launch_pdl(ln_fwd_kernel<32>, dim3(grid), dim3(wpb * 32), 0, stream, xp, M, C, gamma, beta, eps, op, stats));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_layernorm_bwd(const void* dy, const void* x, int M, int C, const float* gamma,
                                 const float* stats, const void* add, void* dx, void* stream_) {
  if (C % 8 != 0 || C > kLnMaxVec * 256) return set_error("layernorm: unsupported C");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int wpb = 8, lpr = ln_lpr(C);
  const int rows_per_block = wpb * (32 / lpr);
  const int grid = (M + rows_per_block - 1) / rows_per_block;
  const bf16 *dyp = reinterpret_cast<const bf16*>(dy), *xp = reinterpret_cast<const bf16*>(x);
  const bf16* ap = reinterpret_cast<const bf16*>(add);
  bf16* dxp = reinterpret_cast<bf16*>(dx);
  if (lpr == 8) CUDA_TRY(launch_pdl(ln_bwd_kernel<8>, dim3(grid), dim3(wpb * 32), 0, stream, dyp, xp, M, C, gamma, stats, ap, dxp));
  else if (lpr == 16) CUDA_TRY(launch_pdl(ln_bwd_kernel<16>, dim3(grid), dim3(wpb * 32), 0, stream, dyp, xp, M, C, gamma, stats, ap, dxp));
  else CUDA_TRY(launch_pdl(ln_bwd_kernel<32>, dim3(grid), dim3(wpb * 32), 0, stream, dyp, xp, M, C, gamma, stats, ap, dxp));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
