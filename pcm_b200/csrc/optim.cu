// Optimiser side of the step on ONE flat fp32 LoRA buffer (67.25 M elements for SD1.5 r=64):
//   pcm_grad_sumsq    : global L2 norm of the (all-reduced) gradient
//   pcm_adamw_clip    : clip_grad_norm_(max_norm) folded into torch.optim.AdamW's update; the
//                       1/world average of the NCCL sum is folded in too; step counter and lr
//                       live in device memory so the whole step can sit in one CUDA graph
//   pcm_lora_refresh  : bf16 operand copies of the LoRA factors in the four layouts the wgmma
//                       GEMMs consume (A, s*B, (s*B)^T, A^T), table driven, one launch
// Replaces accelerator.clip_grad_norm_ + optimizer.step + zero_grad
// (train_pcm_lora_sd15.py:1297-1301) and peft's per-op autocast casts of lora_A / lora_B.
#include "common.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"

namespace pcm {

// out[0] = sum of squares (double).  out[1] is a self-resetting block counter (as uint64), out[2 ..]
// hold one partial per block: the last block to finish adds them in block order, so the norm - and
// with it the clip coefficient and the whole update - is bit-reproducible.
__global__ void sumsq_kernel(const float* __restrict__ g, long long n, double* __restrict__ out) {
  griddep_sync();
  __shared__ double s_part[32];
  __shared__ unsigned long long s_old;
  double acc = 0.0;
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    acc += static_cast<double>(v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (long long i = n4 << 2; i < n; ++i) acc += static_cast<double>(g[i]) * g[i];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < (blockDim.x >> 5) ? s_part[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) {
      out[2 + blockIdx.x] = v;
      __threadfence();
      s_old = atomicAdd(reinterpret_cast<unsigned long long*>(out + 1), 1ULL);
    }
  }
  __syncthreads();
  if (s_old != gridDim.x - 1) return;
  __threadfence();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (unsigned k = 0; k < gridDim.x; ++k) t += __ldcg(out + 2 + k);
    out[0] = t;
    *reinterpret_cast<unsigned long long*>(out + 1) = 0ULL;
  }
}

// state: [0] = lr, [1] = step (float, already incremented for this update)
__global__ void adamw_clip_kernel(float* __restrict__ p, float* __restrict__ g,
                                  float* __restrict__ m, float* __restrict__ v, long long n,
                                  const float* __restrict__ state, float beta1, float beta2,
                                  float eps, float wd, float max_norm, float inv_world,
                                  const double* __restrict__ sumsq, int zero_grad) {
  griddep_sync();
  const float lr = state[0];
  const float step = state[1];
  const float norm = static_cast<float>(sqrt(*sumsq)) * inv_world;
  // torch.nn.utils.clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1
  float coef = max_norm > 0.f ? fminf(max_norm / (norm + 1e-6f), 1.f) : 1.f;
  coef *= inv_world;
  const float bc1 = 1.f - powf(beta1, step);
  const float bc2 = 1.f - powf(beta2, step);
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gi = g[i] * coef;
    float pi = p[i] * (1.f - lr * wd);
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    pi -= step_size * mi / (sqrtf(vi) * inv_sqrt_bc2 + eps);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
    if (zero_grad) g[i] = 0.f;
  }
}

// update_ema (T15:344-355): targ = rate * targ + (1 - rate) * src   (torch: detach().mul_(rate).add_(src, alpha=1-rate))
__global__ void ema_update_kernel(float* __restrict__ targ, const float* __restrict__ src, long long n,
                                  float rate) {
  griddep_sync();
  const float a = 1.f - rate;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    targ[i] = targ[i] * rate + src[i] * a;
}

__global__ void state_step_kernel(float* state) {
  griddep_sync(); state[1] += 1.f; }

// LoRA refresh table entry: masters A [r][taps][cin] and B [n][r] (fp32, offsets in elements)
struct RefreshEntry {
  long long a_off, b_off;              // into the fp32 master buffer
  long long a_fwd, sb_fwd, sb_t, a_t;  // into the bf16 operand buffer
  int cin, taps, n, r;
  long long work_begin;                // prefix sum of per-entry 64x64 tiles (A tiles, then B tiles)
};

// One block per 64x64 fp32 tile (r = 64): coalesced read, bf16 copy in the source layout, and the
// transposed copy through shared memory so both writes are 128-byte contiguous per row.
//   A tile (rows r, columns [c0, c0+64) of tap t): a_fwd[r][t*cin + c]  and  a_t[c][t*64 + r]
//   B tile (rows n0.., columns r):                 sb_fwd[n][r] = s*B   and  sb_t[r][n]
__global__ void __launch_bounds__(256) lora_refresh_kernel(const float* __restrict__ master,
                                                           const RefreshEntry* __restrict__ tab,
                                                           int num_entries, float scale,
                                                           bf16* __restrict__ opnd) {
  griddep_sync();
  __shared__ float tile[64][65];
  __shared__ RefreshEntry e;
  __shared__ long long tidx;
  if (threadIdx.x == 0) {
    const long long i = blockIdx.x;
    int lo = 0, hi = num_entries - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tab[mid].work_begin <= i) lo = mid; else hi = mid - 1;
    }
    e = tab[lo];
    tidx = i - tab[lo].work_begin;
  }
  __syncthreads();
  const int ktot = e.taps * e.cin;
  const long long a_tiles = ktot / 64;
  const bool is_a = tidx < a_tiles;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 float4 columns x 16 rows
  if (is_a) {
    const int c0 = static_cast<int>(tidx) * 64;  // column in [0, taps*cin); one tap per tile
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty + 16 * i;
      const float4 v = *reinterpret_cast<const float4*>(master + e.a_off + static_cast<long long>(r) * ktot + c0 + tx * 4);
      tile[r][tx * 4] = v.x; tile[r][tx * 4 + 1] = v.y; tile[r][tx * 4 + 2] = v.z; tile[r][tx * 4 + 3] = v.w;
      uint2 u;
      u.x = pack_bf16x2(v.x, v.y);
      u.y = pack_bf16x2(v.z, v.w);
      *reinterpret_cast<uint2*>(opnd + e.a_fwd + static_cast<long long>(r) * ktot + c0 + tx * 4) = u;
    }
    __syncthreads();
    const int t = c0 / e.cin, cc0 = c0 - t * e.cin;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = ty + 16 * i;  // a_t row (input channel), 64 consecutive r
      uint2 u;
      u.x = pack_bf16x2(tile[tx * 4][c], tile[tx * 4 + 1][c]);
      u.y = pack_bf16x2(tile[tx * 4 + 2][c], tile[tx * 4 + 3][c]);
      *reinterpret_cast<uint2*>(opnd + e.a_t + (static_cast<long long>(cc0 + c) * e.taps + t) * 64 + tx * 4) = u;
    }
  } else {
    const int n0 = static_cast<int>(tidx - a_tiles) * 64;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int nn = ty + 16 * i;
      float4 v = *reinterpret_cast<const float4*>(master + e.b_off + static_cast<long long>(n0 + nn) * 64 + tx * 4);
      v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
      tile[nn][tx * 4] = v.x; tile[nn][tx * 4 + 1] = v.y; tile[nn][tx * 4 + 2] = v.z; tile[nn][tx * 4 + 3] = v.w;
      uint2 u;
      u.x = pack_bf16x2(v.x, v.y);
      u.y = pack_bf16x2(v.z, v.w);
      *reinterpret_cast<uint2*>(opnd + e.sb_fwd + static_cast<long long>(n0 + nn) * 64 + tx * 4) = u;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty + 16 * i;  // sb_t row, 64 consecutive n
      uint2 u;
      u.x = pack_bf16x2(tile[tx * 4][r], tile[tx * 4 + 1][r]);
      u.y = pack_bf16x2(tile[tx * 4 + 2][r], tile[tx * 4 + 3][r]);
      *reinterpret_cast<uint2*>(opnd + e.sb_t + static_cast<long long>(r) * e.n + n0 + tx * 4) = u;
    }
  }
}

}  // namespace pcm

using namespace pcm;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int pcm_grad_sumsq(const float* g, int64_t n, double* out, void* stream) {
  int grid = static_cast<int>((n / 4 + 255) / 256);
  if (grid > num_sms() * 4) grid = num_sms() * 4;
  if (grid > PCM_SUMSQ_WS_DOUBLES - 2) grid = PCM_SUMSQ_WS_DOUBLES - 2;
  if (grid < 1) grid = 1;
  CUDA_TRY(launch_pdl(sumsq_kernel, dim3(grid), dim3(256), 0, ST(stream), g, n, out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_adamw_clip(float* p, float* g, float* m, float* v, int64_t n, float* state,
                              float beta1, float beta2, float eps, float weight_decay,
                              float max_norm, float inv_world, const double* sumsq, int zero_grad,
                              void* stream) {
  CUDA_TRY(launch_pdl(state_step_kernel, dim3(1), dim3(1), 0, ST(stream), state));
  int grid = static_cast<int>((n + 255) / 256);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  CUDA_TRY(launch_pdl(adamw_clip_kernel, dim3(grid), dim3(256), 0, ST(stream), p, g, m, v, n, state, beta1, beta2, eps,
                                                  weight_decay, max_norm, inv_world, sumsq,
                                                  zero_grad));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_ema_update(float* targ, const float* src, int64_t n, float rate, void* stream) {
  int grid = static_cast<int>((n + 255) / 256);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  if (grid < 1) grid = 1;
  CUDA_TRY(launch_pdl(ema_update_kernel, dim3(grid), dim3(256), 0, ST(stream), targ, src,
                      static_cast<long long>(n), rate));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_lora_refresh(const float* master, const void* table, int num_entries,
                                int64_t total_work, float scale, void* opnd, void* stream) {
  // total_work = number of 64x64 tiles (r must be 64; cin and n multiples of 64)
  CUDA_TRY(launch_pdl(lora_refresh_kernel, dim3(static_cast<unsigned>(total_work)), dim3(256), 0, ST(stream), master, reinterpret_cast<const RefreshEntry*>(table), num_entries, scale,
      reinterpret_cast<bf16*>(opnd)));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
