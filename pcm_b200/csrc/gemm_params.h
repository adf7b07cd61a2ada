// Kernel parameter block of the wgmma implicit-GEMM kernel and its split-K finalize.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "../../include/pcm_b200.h"

namespace pcm {

struct KEntry {
  int a_map, b_map, dw, dh, nchunks, a_c0, b_k0;
  unsigned short n_lo, n_hi;  // n_hi > 0: entry applies to tiles with n_lo <= n0 < n_hi only
  int m_hi;                   // > 0: entry applies to tiles with m0 < m_hi only (its A source has
                              // fewer rows than the output: LoRA T of the leading samples)
  int kend;                   // K columns both operands have from the entry's start:
                              // min(a.C - a_c0, b.K - b_k0); chunk c multiplies min(64, kend - 64c)
                              // of them, rounded up to 16 (narrow kernels only)
};

struct alignas(64) GemmParams {
  CUtensorMap a_maps[PCM_MAX_ASRC];
  CUtensorMap b_maps[PCM_MAX_BSRC];
  KEntry prog[PCM_MAX_PROG];
  int num_prog, lin;
  int M, N;
  int geoW, geoHW;
  int block_n, tiles_m, tiles_n, num_kblocks, num_stages;
  void* out;
  const float* bias;
  const bf16* rowvec;
  const bf16* residual;
  long long osW, osH, osB, rowvec_ld;
  int epiW, epiHW;
  int out_fp32, round_bf16;
  float alpha;
  int act;
  int b_blocked;     // bit i: b_maps[i] is a K-blocked [K/64][N][64] source (3-D map)
  int dep_a_map;     // >= 0: A map written by the previous launch (late PDL wait), -1: none
  int filtered;      // some K entries carry an N range (per-tile K-block count varies)
  int ksplit;        // > 1: work item = (tile, K split); split s stores its fp32 partial sums to
  float* ws;         // ws[s][m * N + n]; the finalize kernel adds the slices in order and applies
                     // bias / residual / activation
};

constexpr int kATileBytes = 128 * 128;  // 128 rows x 64 bf16

}  // namespace pcm
