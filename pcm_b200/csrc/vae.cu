// Glue kernels of the Stable Diffusion VAE (AutoencoderKL) around the implicit GEMM: the mid-block
// attention's row softmax and V transpose, the latent distribution after the encoder, the decoder's
// entry (post_quant_conv) and the image exit.
//
// Replaces, in diffusers' AutoencoderKL as the reference calls it (T15:1127-1136 vae.encode(...)
// .latent_dist.sample(), log_validation's pipeline vae.decode): Attention.get_attention_scores'
// softmax, DiagonalGaussianDistribution, post_quant_conv and VaeImageProcessor.postprocess.
#include "common.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"

namespace pcm {

constexpr int kSoftmaxThreads = 256;

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();   // red is reused by the next reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < kSoftmaxThreads / 32; ++w) v = is_max ? fmaxf(v, red[w]) : v + red[w];
  return v;
}

// p[r, :] = bf16(exp(s[r, :] - max) / sum exp(s[r, :] - max)), fp32 max and sum; one block per row, the
// row read three times (max, sum, store; it stays in L2).  Fixed reduction order: reproducible.
__global__ void __launch_bounds__(kSoftmaxThreads) softmax_rows_kernel(const float* __restrict__ s, int cols,
                                                                       long long lds, bf16* __restrict__ p,
                                                                       long long ldp) {
  griddep_sync();
  __shared__ float red[kSoftmaxThreads / 32];
  const float4* row = reinterpret_cast<const float4*>(s + blockIdx.x * lds);
  const int nv = cols >> 2;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < nv; i += kSoftmaxThreads) {
    const float4 x = row[i];
    m = fmaxf(m, fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w)));
  }
  m = block_reduce(m, true, red);
  float sum = 0.f;
  for (int i = threadIdx.x; i < nv; i += kSoftmaxThreads) {
    const float4 x = row[i];
    sum += (expf(x.x - m) + expf(x.y - m)) + (expf(x.z - m) + expf(x.w - m));
  }
  sum = block_reduce(sum, false, red);
  const float inv = 1.f / sum;
  uint2* out = reinterpret_cast<uint2*>(p + blockIdx.x * ldp);
  for (int i = threadIdx.x; i < nv; i += kSoftmaxThreads) {
    const float4 x = row[i];
    out[i] = make_uint2(pack_bf16x2(expf(x.x - m) * inv, expf(x.y - m) * inv),
                        pack_bf16x2(expf(x.z - m) * inv, expf(x.w - m) * inv));
  }
}

// out[b][c][r] = in[b][r][c] for a batch of bf16 [rows, cols] matrices (32 x 32 tiles through shared memory)
__global__ void transpose_bf16_kernel(const uint16_t* __restrict__ in, int rows, int cols, long long ldi,
                                      long long bsi, uint16_t* __restrict__ out, long long ldo, long long bso) {
  griddep_sync();
  __shared__ uint16_t t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  in += blockIdx.z * bsi;
  out += blockIdx.z * bso;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) t[j][threadIdx.x] = in[r * ldi + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[c * ldo + r] = t[threadIdx.x][j];
  }
}

// quant_conv (1x1, 8 -> 8) on h [B*HW, 8] and DiagonalGaussianDistribution: moments rounded to bf16 like
// the conv's output, logvar clamped to [-30, 20], std = exp(logvar / 2); NCHW [B, 4, HW] outputs.  With noise
// (NCHW [B, 4, HW]): sample = (mean + std * noise) * scale, each operation rounded on its own as torch does.
__global__ void latent_dist_kernel(const float* __restrict__ h, int B, int HW, const bf16* __restrict__ w,
                                   const float* __restrict__ bias, const float* __restrict__ noise, float scale,
                                   float* __restrict__ mean, float* __restrict__ logvar, float* __restrict__ stdv,
                                   float* __restrict__ sample) {
  griddep_sync();
  const long long total = static_cast<long long>(B) * HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / HW, px = i - b * HW;
    float x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = __bfloat162float(__float2bfloat16_rn(h[i * 8 + k]));
    float mo[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) acc = fmaf(x[k], __bfloat162float(w[o * 8 + k]), acc);
      mo[o] = __bfloat162float(__float2bfloat16_rn(acc + bias[o]));
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const long long o = (b * 4 + c) * HW + px;
      const float lv = fminf(fmaxf(mo[4 + c], -30.f), 20.f);
      const float sd = expf(0.5f * lv);
      mean[o] = mo[c];
      logvar[o] = lv;
      stdv[o] = sd;
      if (noise) sample[o] = __fmul_rn(__fadd_rn(mo[c], __fmul_rn(sd, noise[o])), scale);
    }
  }
}

// post_quant_conv (1x1, 4 -> 4) on z / div: fp32 NHWC [M, 4] in, bf16 NHWC [M, 8] out, channels 4..7 zero (the
// A source of the decoder's conv_in on the implicit GEMM: 16-byte pixels, as TMA needs)
__global__ void vae_dec_in_kernel(const float* __restrict__ z, long long M, const bf16* __restrict__ w,
                                  const float* __restrict__ bias, float div, bf16* __restrict__ out) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < M;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = *reinterpret_cast<const float4*>(z + i * 4);
    const float x[4] = {__bfloat162float(__float2bfloat16_rn(__fdiv_rn(v.x, div))),
                        __bfloat162float(__float2bfloat16_rn(__fdiv_rn(v.y, div))),
                        __bfloat162float(__float2bfloat16_rn(__fdiv_rn(v.z, div))),
                        __bfloat162float(__float2bfloat16_rn(__fdiv_rn(v.w, div)))};
    float y[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) acc = fmaf(x[k], __bfloat162float(w[o * 4 + k]), acc);
      y[o] = acc + bias[o];
    }
    *reinterpret_cast<uint4*>(out + i * 8) = make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), 0u, 0u);
  }
}

// (x / 2 + 0.5).clamp(0, 1): fp32 NHWC [B, HW, C] in, fp32 NCHW out, and optionally uint8 NHWC
// round(v * 255) (round half to even, as numpy's round)
__global__ void image_exit_kernel(const float* __restrict__ x, int B, int HW, int C, float* __restrict__ out,
                                  uint8_t* __restrict__ u8) {
  griddep_sync();
  const long long total = static_cast<long long>(B) * HW * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long px = i / C;
    const int c = static_cast<int>(i - px * C);
    const long long b = px / HW, p = px - b * HW;
    const float v = fminf(fmaxf(__fadd_rn(x[i] * 0.5f, 0.5f), 0.f), 1.f);
    if (out) out[(b * C + c) * HW + p] = v;
    if (u8) u8[i] = static_cast<uint8_t>(rintf(__fmul_rn(v, 255.f)));
  }
}

static inline int vae_grid(long long total, int threads) {
  long long g = (total + threads - 1) / threads;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

static bool unaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

}  // namespace pcm

using namespace pcm;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int pcm_softmax_rows(const float* s, int64_t rows, int cols, int64_t lds, void* p, int64_t ldp,
                                void* stream) {
  if (rows < 1 || rows > 2147483647LL) return set_error("softmax_rows: rows must be in [1, 2^31)");
  if (cols < 4 || cols % 4 != 0) return set_error("softmax_rows: cols must be a positive multiple of 4");
  if (lds % 4 != 0 || ldp % 4 != 0 || lds < cols || ldp < cols)
    return set_error("softmax_rows: lds and ldp must be multiples of 4, at least cols");
  if (unaligned(s, 16) || unaligned(p, 8)) return set_error("softmax_rows: s must be 16-byte, p 8-byte aligned");
  CUDA_TRY(launch_pdl(softmax_rows_kernel, dim3(static_cast<unsigned>(rows)), dim3(kSoftmaxThreads), 0, ST(stream),
                      s, cols, static_cast<long long>(lds), reinterpret_cast<bf16*>(p), static_cast<long long>(ldp)));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_transpose_bf16(const void* in, int rows, int cols, int64_t ldi, int64_t bsi, int batch,
                                  void* out, int64_t ldo, int64_t bso, void* stream) {
  if (rows < 1 || cols < 1 || batch < 1 || batch > 65535) return set_error("transpose_bf16: bad shape");
  if (ldi < cols || ldo < rows) return set_error("transpose_bf16: ldi must be >= cols, ldo >= rows");
  dim3 grid((cols + 31) / 32, (rows + 31) / 32, batch);
  if (grid.y > 65535) return set_error("transpose_bf16: too many rows");
  CUDA_TRY(launch_pdl(transpose_bf16_kernel, grid, dim3(32, 8), 0, ST(stream), reinterpret_cast<const uint16_t*>(in),
                      rows, cols, static_cast<long long>(ldi), static_cast<long long>(bsi),
                      reinterpret_cast<uint16_t*>(out), static_cast<long long>(ldo), static_cast<long long>(bso)));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_latent_dist(const float* h, int B, int HW, const void* w, const float* bias, const float* noise,
                               float scale, float* mean, float* logvar, float* std, float* sample, void* stream) {
  if (B < 1 || HW < 1) return set_error("latent_dist: bad shape");
  if (noise && !sample) return set_error("latent_dist: noise without sample");
  const long long total = static_cast<long long>(B) * HW;
  CUDA_TRY(launch_pdl(latent_dist_kernel, dim3(vae_grid(total, 256)), dim3(256), 0, ST(stream), h, B, HW,
                      reinterpret_cast<const bf16*>(w), bias, noise, scale, mean, logvar, std, sample));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_vae_dec_in(const float* z, int64_t M, const void* w, const float* bias, float div, void* out,
                              void* stream) {
  if (M < 1) return set_error("vae_dec_in: M must be >= 1");
  if (unaligned(z, 16) || unaligned(out, 16)) return set_error("vae_dec_in: z and out must be 16-byte aligned");
  CUDA_TRY(launch_pdl(vae_dec_in_kernel, dim3(vae_grid(M, 256)), dim3(256), 0, ST(stream), z,
                      static_cast<long long>(M), reinterpret_cast<const bf16*>(w), bias, div, reinterpret_cast<bf16*>(out)));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_image_exit(const float* x, int B, int HW, int C, float* out, void* u8, void* stream) {
  if (B < 1 || HW < 1 || C < 1) return set_error("image_exit: bad shape");
  const long long total = static_cast<long long>(B) * HW * C;
  CUDA_TRY(launch_pdl(image_exit_kernel, dim3(vae_grid(total, 256)), dim3(256), 0, ST(stream), x, B, HW, C, out,
                      reinterpret_cast<uint8_t*>(u8)));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
