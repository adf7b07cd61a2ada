// pcm_lora_fuse: LoRA fused into the frozen weights for inference (peft `fuse_lora`, which the
// reference's validation pipeline calls before sampling, T15:120-207):
//   W_out[n, k] = bf16( float(W_in[n, k]) + scale * sum_r B[n, r] * A[r, k] )
// on the K-blocked [K/64][N_total][64] bf16 layout the GEMMs read, out of place (the trained network's
// frozen weights are only read).  A / B come from the fp32 LoRA masters (`lora_master` or any flat
// buffer of the same layout).  The rank sum runs in fp32 in ascending rank order and the result is
// rounded to bf16 once, so repeated fusions are bitwise identical.
//
// SIMT FP32: one 256-thread block per 64 (rows) x 64 (K columns) output tile; each thread owns a 4 x 4
// sub-tile, ranks are staged through shared memory 32 at a time (A as [rank][k], B transposed to
// [rank][n]) so the inner loop is two float4 loads per 16 FMAs.
#include "common.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"

namespace pcm {

struct FuseEntry {
  long long a_off, b_off;   // A [r][K] and B [n][r] in the fp32 master buffer (elements)
  long long src, dst;       // K-blocked bf16 operands [K/64][N_total][64] (device addresses)
  long long n0_ntot;        // row offset of the layer inside the stacked operand | N_total << 32
  long long k_r;            // K = taps * cin | r << 32
  long long n;              // the layer's rows (output channels)
  long long work_begin;     // prefix sum of 64 x 64 tiles: (n / 64) * (K / 64) per entry
};

constexpr int kFuseRC = 32;   // ranks per shared-memory stage

__global__ void __launch_bounds__(256) lora_fuse_kernel(const float* __restrict__ master,
                                                        const FuseEntry* __restrict__ tab,
                                                        int num_entries, float scale) {
  griddep_sync();
  __shared__ __align__(16) float As[kFuseRC][64];
  __shared__ __align__(16) float Bs[kFuseRC][68];
  __shared__ FuseEntry e;
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
  const int K = static_cast<int>(e.k_r & 0xffffffffLL), r = static_cast<int>(e.k_r >> 32);
  const int n0 = static_cast<int>(e.n0_ntot & 0xffffffffLL);
  const long long ntot = e.n0_ntot >> 32;
  const int n_tiles = static_cast<int>(e.n / 64);
  const int nt = static_cast<int>(tidx % n_tiles), kt = static_cast<int>(tidx / n_tiles);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // k = 4 tx + j, n = 4 ty + i
  const float* A = master + e.a_off + 64LL * kt;            // A[rank][64 kt + c] at rank * K + c
  const float* B = master + e.b_off + 64LL * nt * r;        // B[64 nt + n][rank] at n * r + rank
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int r0 = 0; r0 < r; r0 += kFuseRC) {
    const int rc = min(kFuseRC, r - r0);                     // a multiple of 8
    // A stage: rc rows of 64 floats (16 float4 per row)
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const int q = threadIdx.x + 256 * p, row = q >> 4, c4 = q & 15;
      if (row < rc)
        *reinterpret_cast<float4*>(&As[row][c4 * 4]) =
            *reinterpret_cast<const float4*>(A + static_cast<long long>(r0 + row) * K + c4 * 4);
    }
    // B stage: 64 rows of rc floats, stored transposed
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const int q = threadIdx.x + 256 * p, nn = q >> 3, c4 = q & 7;
      if (c4 * 4 < rc) {
        const float4 v = *reinterpret_cast<const float4*>(B + static_cast<long long>(nn) * r + r0 + c4 * 4);
        Bs[c4 * 4][nn] = v.x; Bs[c4 * 4 + 1][nn] = v.y; Bs[c4 * 4 + 2][nn] = v.z; Bs[c4 * 4 + 3][nn] = v.w;
      }
    }
    __syncthreads();
    for (int j = 0; j < rc; ++j) {
      const float4 a = *reinterpret_cast<const float4*>(&As[j][tx * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[j][ty * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) acc[i][jj] = __fmaf_rn(bv[i], av[jj], acc[i][jj]);
    }
    __syncthreads();
  }
  const bf16* src = reinterpret_cast<const bf16*>(e.src);
  bf16* dst = reinterpret_cast<bf16*>(e.dst);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long off = (static_cast<long long>(kt) * ntot + n0 + 64LL * nt + ty * 4 + i) * 64 + tx * 4;
    const uint2 w = *reinterpret_cast<const uint2*>(src + off);
    const bf16* wv = reinterpret_cast<const bf16*>(&w);
    float o[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
      o[jj] = __fadd_rn(__bfloat162float(wv[jj]), __fmul_rn(scale, acc[i][jj]));
    uint2 u;
    u.x = pack_bf16x2(o[0], o[1]);
    u.y = pack_bf16x2(o[2], o[3]);
    *reinterpret_cast<uint2*>(dst + off) = u;
  }
}

}  // namespace pcm

using namespace pcm;

extern "C" int pcm_lora_fuse(const float* master, const void* table, int num_entries, int64_t total_work,
                             float scale, void* stream) {
  if (num_entries < 1 || total_work < 1) return set_error("pcm_lora_fuse: empty table");
  CUDA_TRY(launch_pdl(lora_fuse_kernel, dim3(static_cast<unsigned>(total_work)), dim3(256), 0,
                      reinterpret_cast<cudaStream_t>(stream), master,
                      reinterpret_cast<const FuseEntry*>(table), num_entries, scale));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
