// wgmma / TMA implicit-GEMM for sm_90a.
//
//   pcm_gemm  : out[M, N] = alpha * sum_k A[m, k] * Bw[n, k]  (+bias, +per-image row vector,
//               +residual, optional SiLU).  A is gathered by TMA from up to 6 NHWC bf16 tensors
//               through a "K program" (spatial taps x channel chunks x K segments), so the same
//               kernel runs nn.Linear, 1x1 / 3x3 / stride-2 convolutions (parity planes),
//               skip-concat convolutions (two K segments), the LoRA up-projection fused as an
//               extra 64-wide K segment, and all of their dgrads (taps mirrored, W transposed).
//   pcm_wgrad : out[ch, r] += alpha * sum_m P[m(+tap), ch] * Q[m, r]   (LoRA A/B weight grads),
//               both operands MN-major straight from the activation layout, split over tokens.
//
// Replaces the cuDNN / cuBLAS calls that diffusers' UNet2DConditionModel + peft LoRA issue for
// train_pcm_lora_sd15.py:1192-1198, 1219-1223, 1238-1244, 1263-1268 (forwards) and :1296
// (backward).  Warpgroup roles: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 =
// consumers, each owning 64 rows of the 128 x BN output tile: wgmma into registers, then the
// epilogue from those registers (gemm_epilogue.cuh) while the producer already fills the stages of
// the next tile.  BN (the N tile, a multiple of 32 up to 256) is a template parameter: it is the N
// of the wgmma instruction.
// K-program entries may be restricted to an output-column range (grouped Linear layers sharing
// their input) or to the leading M tiles (an A source with fewer rows than the output: the LoRA
// T of the student samples in the merged student + teacher pass).  Weights may be K-blocked
// ([K/64][N][64], pcm_bsrc.kblocked).  dep_a_src1: late programmatic-dependent-launch wait on the
// LoRA down-projection, M tiles visited last-to-first.  split-K: ordered workspace slices + finalize.
#include "common.cuh"
#include "wgmma.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"
#include "gemm_params.h"
#include "gemm_epilogue.cuh"

namespace pcm {

constexpr int kGemmThreads = 384;   // warpgroup 0 TMA, warpgroups 1-2 wgmma + epilogue
constexpr int kWgradThreads = 256;  // warpgroup 0 TMA, warpgroup 1 wgmma + reduction
constexpr int kMaxStages = 8;
constexpr int kStagingBytes = 2 * 64 * 32 * 4;   // epilogue transposition buffers (fp32), one per consumer
constexpr int kSmemLimit = 227 * 1024 - 512;     // dynamic smem budget (227 KB max minus static)

// K blocks of the work item whose output tile starts at rows m0, columns n0 (filtered programs)
__device__ __forceinline__ int tile_kblocks(const GemmParams& p, int m0, int n0) {
  int nkb = 0;
  for (int e = 0; e < p.num_prog; ++e) {
    const KEntry en = p.prog[e];
    if ((en.n_hi == 0 || (n0 >= en.n_lo && n0 < en.n_hi)) && (en.m_hi == 0 || m0 < en.m_hi))
      nkb += en.nchunks;
  }
  return nkb;
}

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
pcm_gemm_kernel(const __grid_constant__ GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];

  const int wg = threadIdx.x >> 7;
  const int S = p.num_stages;
  constexpr uint32_t stage_bytes = kATileBytes + BN * 128;
  const int num_items = p.tiles_m * p.tiles_n * p.ksplit;
  const int kb_per = (p.num_kblocks + p.ksplit - 1) / p.ksplit;

  if (threadIdx.x == 0) {
    for (int i = 0; i < PCM_MAX_ASRC; ++i) tma_prefetch_desc(&p.a_maps[i]);
    for (int i = 0; i < PCM_MAX_BSRC; ++i) tma_prefetch_desc(&p.b_maps[i]);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: everything above overlapped the previous kernel's tail.  With a late dependency
  // (dep_a_map >= 0: only the LoRA down-projection T comes from the previous launch, everything else
  // from launches that one has already waited for) the base K blocks start right away and only the
  // TMA producer waits, just before its first read of T.
  if (p.dep_a_map < 0) griddep_sync();
  else griddep_launch();

  if (wg == 0) {
    // ===================== TMA producer =====================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      bool dep_waited = p.dep_a_map < 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int tile = item / p.ksplit, ks = item - tile * p.ksplit;
        const int kb0 = ks * kb_per, kb1 = min(p.num_kblocks, kb0 + kb_per);
        int tm = tile / p.tiles_n;
        const int tn = tile - tm * p.tiles_n;
        if (p.dep_a_map >= 0) tm = p.tiles_m - 1 - tm;  // adapter-free rows first (see dep_a_src1)
        const int m0 = tm * 128, n0 = tn * BN;
        int b0 = 0, h0 = 0;
        if (!p.lin) {
          b0 = m0 / p.geoHW;
          h0 = (m0 - b0 * p.geoHW) / p.geoW;
        }
        int kidx = 0;
        for (int e = 0; e < p.num_prog; ++e) {
          const KEntry en = p.prog[e];
          if (en.n_hi != 0 && (n0 < en.n_lo || n0 >= en.n_hi)) continue;  // other layer's K block
          if (en.m_hi != 0 && m0 >= en.m_hi) continue;  // rows past the end of this entry's A source
          if (kidx + en.nchunks <= kb0 || kidx >= kb1) {  // entry entirely outside this K split
            kidx += en.nchunks;
            continue;
          }
          if (!dep_waited && en.a_map == p.dep_a_map) {
            griddep_wait();  // the previous launch (T = x A^T) is complete and visible
            dep_waited = true;
          }
          for (int c = 0; c < en.nchunks; ++c, ++kidx) {
            if (kidx < kb0 || kidx >= kb1) continue;
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
            uint8_t* sa = smem + stage * stage_bytes;
            uint8_t* sb = sa + kATileBytes;
            if (p.lin)
              tma_load_4d(sa, &p.a_maps[en.a_map], &full_bar[stage], en.a_c0 + c * 64, m0, 0, 0);
            else
              tma_load_4d(sa, &p.a_maps[en.a_map], &full_bar[stage], en.a_c0 + c * 64, en.dw,
                          h0 + en.dh, b0);
            if ((p.b_blocked >> en.b_map) & 1)   // K-blocked weights: (64, N, K/64) view, contiguous tile
              tma_load_3d(sb, &p.b_maps[en.b_map], &full_bar[stage], 0, n0, (en.b_k0 >> 6) + c);
            else
              tma_load_2d(sb, &p.b_maps[en.b_map], &full_bar[stage], en.b_k0 + c * 64, n0);
            if (++stage == S) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma mainloop + epilogue =====================
    regs_alloc<232>();   // 128 x 40 + 256 x 232 <= 64 K registers
    const int cw = wg - 1;                 // rows cw * 64 .. cw * 64 + 63 of the tile
    const int et = threadIdx.x & 127;
    float* sbuf = reinterpret_cast<float*>(smem + S * stage_bytes) + cw * (64 * 32);
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const int tile = item / p.ksplit, ks = item - tile * p.ksplit;
      int tm = tile / p.tiles_n;
      const int tn = tile - tm * p.tiles_n;
      if (p.dep_a_map >= 0) tm = p.tiles_m - 1 - tm;
      const int n0 = tn * BN;
      const int nkb = p.filtered ? tile_kblocks(p, tm * 128, n0)   // N- or M-ranged entries (ksplit == 1)
                                 : min(p.num_kblocks, (ks + 1) * kb_per) - ks * kb_per;
      if (nkb <= 0) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      }
      int prev_stage = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * stage_bytes) + cw * (64 * 128);
        const uint32_t b_addr = smem_u32(smem + stage * stage_bytes) + kATileBytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<BN, 0, 0>::mma(acc, wgmma_desc_sw128(a_addr + k * 32, 16, 1024),
                               wgmma_desc_sw128(b_addr + k * 32, 16, 1024), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_fence_acc(acc);
        // the previous K block's wgmma are complete: its stage may be refilled
        wgmma_wait<1>();
        if (prev_stage >= 0 && et == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == S) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (prev_stage >= 0 && et == 0) mbar_arrive(&empty_bar[prev_stage]);
      // split-K: this item's partial sums go to slice ks of the workspace
      float* ws = p.ws ? p.ws + static_cast<long long>(ks) * p.M * p.N : nullptr;
      gemm_epilogue_tile<BN>(p, tm * 128 + cw * 64, n0, acc, sbuf, et, 1 + cw, ws);
    }
  }
}

// split-K finalize: out = act(sum over the ksplit workspace slices, in split order, + bias + rowvec
// + residual), same row mapping as the GEMM epilogue.  Fixed summation order: reproducible.
__global__ void splitk_finalize_kernel(const GemmParams p) {
  griddep_sync();
  const int nvec = (p.N + 7) >> 3;
  const long long total = static_cast<long long>(p.M) * nvec;
  const long long slice = static_cast<long long>(p.M) * p.N;
  const bool vec = (p.N & 7) == 0;   // 8 consecutive columns per thread: two 16-byte loads per slice
  for (long long v = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; v < total;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(v / nvec);
    const int n = static_cast<int>(v - static_cast<long long>(m) * nvec) * 8;
    const int b = m / p.epiHW;
    const int r = m - b * p.epiHW;
    const int h = r / p.epiW;
    const int w = r - h * p.epiW;
    const long long o = b * p.osB + h * p.osH + w * p.osW;
    float x[8];
    const float* wp = p.ws + static_cast<long long>(m) * p.N + n;
    if (vec) {
      float4 a0 = *reinterpret_cast<const float4*>(wp), a1 = *reinterpret_cast<const float4*>(wp + 4);
#pragma unroll 4
      for (int k = 1; k < p.ksplit; ++k) {   // split order: reproducible (loads of 4 slices in flight)
        const float4 b0 = *reinterpret_cast<const float4*>(wp + k * slice);
        const float4 b1 = *reinterpret_cast<const float4*>(wp + k * slice + 4);
        a0.x += b0.x; a0.y += b0.y; a0.z += b0.z; a0.w += b0.w;
        a1.x += b1.x; a1.y += b1.y; a1.z += b1.z; a1.w += b1.w;
      }
      x[0] = a0.x; x[1] = a0.y; x[2] = a0.z; x[3] = a0.w;
      x[4] = a1.x; x[5] = a1.y; x[6] = a1.z; x[7] = a1.w;
    } else {
      for (int e = 0; e < 8; ++e) {
        x[e] = 0.f;
        if (n + e < p.N) {
          x[e] = wp[e];
          for (int k = 1; k < p.ksplit; ++k) x[e] += wp[k * slice + e];
        }
      }
    }
    for (int e = 0; e < 8 && n + e < p.N; ++e) {
      float y = x[e];
      if (p.bias) y += p.bias[n + e];
      if (p.rowvec) y += __bfloat162float(p.rowvec[b * p.rowvec_ld + n + e]);
      if (p.residual) y += __bfloat162float(p.residual[o + n + e]);
      if (p.act == 1) y = silu_f(y);
      if (p.out_fp32) {
        if (p.round_bf16) y = __bfloat162float(__float2bfloat16_rn(y));
        reinterpret_cast<float*>(p.out)[o + n + e] = y;
      } else {
        reinterpret_cast<bf16*>(p.out)[o + n + e] = __float2bfloat16_rn(y);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// LoRA weight gradient: out[ch, r] += alpha * sum_tokens P[tok(+tap), ch] * Q[tok, r]
// ------------------------------------------------------------------------------------------
struct alignas(64) WgradParams {
  CUtensorMap p_map;
  CUtensorMap q_map;
  int lin, geoW, geoHW;
  int M, Cp, q_c0;
  int num_taps;
  int dw[9], dh[9];
  long long tap_off[9];
  int ksplit, kblocks_total;
  float* out;
  long long os_row, os_col;
  float alpha;
  int* sem;  // deterministic mode: one turnstile per (channel tile, tap); NULL = unordered atomics
};

constexpr int kWgStages = 4;
constexpr int kWgStageBytes = 3 * kATileBytes;  // P: 2 x (128 tok x 64 ch), Q: 128 tok x 64 r

__global__ void __launch_bounds__(kWgradThreads, 1)
pcm_wgrad_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  __shared__ __align__(8) uint64_t full_bar[kWgStages];
  __shared__ __align__(8) uint64_t empty_bar[kWgStages];

  const int ch0 = blockIdx.x * 128;
  const int tap = blockIdx.y;
  const int per = (p.kblocks_total + p.ksplit - 1) / p.ksplit;
  const int kb_begin = blockIdx.z * per;
  const int kb_end = min(p.kblocks_total, kb_begin + per);
  const int nkb = kb_end - kb_begin;
  if (nkb <= 0) return;  // uniform per CTA

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.p_map);
    tma_prefetch_desc(&p.q_map);
    for (int i = 0; i < kWgStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_sync();  // PDL: everything above overlapped the previous kernel's tail

  if (threadIdx.x < 128) {
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        const int m0 = kb * 128;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], kWgStageBytes);
        uint8_t* sp = smem + stage * kWgStageBytes;
        uint8_t* sq = sp + 2 * kATileBytes;
        if (p.lin) {
          tma_load_4d(sp, &p.p_map, &full_bar[stage], ch0, m0, 0, 0);
          tma_load_4d(sp + kATileBytes, &p.p_map, &full_bar[stage], ch0 + 64, m0, 0, 0);
          tma_load_4d(sq, &p.q_map, &full_bar[stage], p.q_c0, m0, 0, 0);
        } else {
          const int b0 = m0 / p.geoHW;
          const int h0 = (m0 - b0 * p.geoHW) / p.geoW;
          tma_load_4d(sp, &p.p_map, &full_bar[stage], ch0, p.dw[tap], h0 + p.dh[tap], b0);
          tma_load_4d(sp + kATileBytes, &p.p_map, &full_bar[stage], ch0 + 64, p.dw[tap],
                      h0 + p.dh[tap], b0);
          tma_load_4d(sq, &p.q_map, &full_bar[stage], p.q_c0, 0, h0, b0);
        }
        if (++stage == kWgStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // two m64 n64 accumulators: channels ch0 .. ch0 + 63 (P tile 0) and ch0 + 64 .. (P tile 1)
    const int et = threadIdx.x & 127;
    float acc0[32], acc1[32];
    int stage = 0;
    uint32_t phase = 0;
    int prev_stage = -1;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t p_addr = smem_u32(smem + stage * kWgStageBytes);
      const uint32_t q_addr = p_addr + 2 * kATileBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {  // 16 tokens per wgmma
        const uint64_t bd = wgmma_desc_sw128(q_addr + k * 2048, kATileBytes, 1024);
        const uint32_t accum = (i | k) != 0 ? 1u : 0u;
        Wgmma<64, 1, 1>::mma(acc0, wgmma_desc_sw128(p_addr + k * 2048, kATileBytes, 1024), bd, accum);
        Wgmma<64, 1, 1>::mma(acc1, wgmma_desc_sw128(p_addr + kATileBytes + k * 2048, kATileBytes, 1024), bd,
                             accum);
      }
      wgmma_commit();
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
      wgmma_wait<1>();
      if (prev_stage >= 0 && et == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == kWgStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc0);
    wgmma_fence_acc(acc1);
    // Deterministic mode: the token splits of one output tile add their partial sums in split
    // order (turnstile on a per-tile semaphore).  Lower blockIdx.z CTAs are dispatched first and
    // never wait on higher ones, so the chain cannot deadlock.
    int* sem = p.sem ? p.sem + (blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
    if (sem) {
      if (et == 0) {
        while (atomicAdd(sem, 0) != static_cast<int>(blockIdx.z)) __nanosleep(64);
        __threadfence();
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    // fragment rows (channels) 16 (et / 32) + (et % 32) / 4 (+8), columns (ranks) 8 q + 2 (et % 4) (+1)
    const int frow = ((et >> 5) << 4) + ((et & 31) >> 2);
    const int fcol = 2 * (et & 3);
    const float* o_base = p.out + p.tap_off[tap];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const float* acc = hf ? acc1 : acc0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ch = ch0 + hf * 64 + frow + 8 * h;
        if (ch >= p.Cp) continue;
        float* o = const_cast<float*>(o_base) + static_cast<long long>(ch) * p.os_row;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int r = 8 * q + fcol;
          const float v0 = acc[4 * q + 2 * h] * p.alpha, v1 = acc[4 * q + 2 * h + 1] * p.alpha;
          if (p.os_col == 1) {   // rank index contiguous (dB layout [n][r]): 8-byte vector reductions
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(o + r), "f"(v0), "f"(v1) : "memory");
          } else {
            atomicAdd(o + static_cast<long long>(r) * p.os_col, v0);
            atomicAdd(o + static_cast<long long>(r + 1) * p.os_col, v1);
          }
        }
      }
    }
    if (sem) {
      __threadfence();
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (et == 0)
        atomicExch(sem, blockIdx.z + 1 == gridDim.z ? 0 : static_cast<int>(blockIdx.z) + 1);
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static int encode_asrc(CUtensorMap* map, const pcm_asrc& a, int lin, int geoW, int geoH,
                       int box_c = 64) {
  cuuint64_t dims[4];
  cuuint64_t strides[3];
  cuuint32_t box[4];
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (lin) {
    // [rows = a.W, C] matrix; box = 64 x 128 rows
    dims[0] = a.C; dims[1] = a.W; dims[2] = 1; dims[3] = 1;
    strides[0] = a.sW * 2;
    strides[1] = static_cast<cuuint64_t>(a.sW) * 2 * a.W;
    strides[2] = strides[1];
    box[0] = box_c; box[1] = 128; box[2] = 1; box[3] = 1;
  } else {
    dims[0] = a.C; dims[1] = a.W; dims[2] = a.H; dims[3] = a.B;
    strides[0] = a.sW * 2; strides[1] = a.sH * 2; strides[2] = a.sB * 2;
    const int bw = geoW;
    if (bw > 128 || 128 % bw != 0) return set_error("conv geometry: W must divide 128");
    int bh = 128 / bw;
    if (bh > geoH) bh = geoH;
    int bb = 128 / (bw * bh);
    if (bw * bh * bb != 128) return set_error("conv geometry: H*W must divide or be divisible by 128");
    box[0] = box_c; box[1] = bw; box[2] = bh; box[3] = bb;
  }
  return encode_tmap(map, a.ptr, 4, dims, strides, box, estr);
}

// the wgmma N of the kernel is the N tile of the launch
typedef void (*GemmKernel)(const GemmParams);
static GemmKernel gemm_kernel_for(int block_n) {
  switch (block_n) {
    case 32: return pcm_gemm_kernel<32>;
    case 64: return pcm_gemm_kernel<64>;
    case 96: return pcm_gemm_kernel<96>;
    case 128: return pcm_gemm_kernel<128>;
    case 160: return pcm_gemm_kernel<160>;
    case 192: return pcm_gemm_kernel<192>;
    case 224: return pcm_gemm_kernel<224>;
    default: return pcm_gemm_kernel<256>;
  }
}

static int launch_gemm(const pcm_gemm_desc* d, cudaStream_t stream) {
  if (d->block_n < 32 || d->block_n > 256 || (d->block_n % 32) != 0)
    return set_error("pcm_gemm: block_n must be a multiple of 32 in [32, 256]");
  if (d->num_a < 1 || d->num_a > PCM_MAX_ASRC || d->num_b < 1 || d->num_b > PCM_MAX_BSRC ||
      d->num_prog < 1 || d->num_prog > PCM_MAX_PROG)
    return set_error("pcm_gemm: bad source / program counts");
  static GemmParams p;  // host staging (single host thread per rank)
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < PCM_MAX_ASRC; ++i) {
    const pcm_asrc& a = d->a[i < d->num_a ? i : 0];
    if (int rc = encode_asrc(&p.a_maps[i], a, d->lin, d->geoW, d->geoH)) return rc;
  }
  for (int i = 0; i < PCM_MAX_BSRC; ++i) {
    const pcm_bsrc& b = d->b[i < d->num_b ? i : 0];
    if (b.kblocked) {   // [K/64][N][64]: 3-D view (k within block, n, K block)
      if (b.K % 64 != 0) return set_error("pcm_gemm: K-blocked B source needs K % 64 == 0");
      cuuint64_t dims[3] = {64, static_cast<cuuint64_t>(b.N), static_cast<cuuint64_t>(b.K / 64)};
      cuuint64_t strides[2] = {128, static_cast<cuuint64_t>(b.N) * 128};
      cuuint32_t box[3] = {64, static_cast<cuuint32_t>(d->block_n), 1};
      cuuint32_t estr[3] = {1, 1, 1};
      if (int rc = encode_tmap(&p.b_maps[i], b.ptr, 3, dims, strides, box, estr)) return rc;
      if (i < d->num_b) p.b_blocked |= 1 << i;
    } else {
      cuuint64_t dims[2] = {static_cast<cuuint64_t>(b.K), static_cast<cuuint64_t>(b.N)};
      cuuint64_t strides[1] = {static_cast<cuuint64_t>(b.ld) * 2};
      cuuint32_t box[2] = {64, static_cast<cuuint32_t>(d->block_n)};
      cuuint32_t estr[2] = {1, 1};
      if (int rc = encode_tmap(&p.b_maps[i], b.ptr, 2, dims, strides, box, estr)) return rc;
    }
  }
  int nkb = 0;
  for (int e = 0; e < d->num_prog; ++e) {
    const pcm_kentry& k = d->prog[e];
    if (k.a_src < 0 || k.a_src >= d->num_a || k.b_src < 0 || k.b_src >= d->num_b || k.nchunks < 1 ||
        (k.b_k0 & 63) != 0)
      return set_error("pcm_gemm: bad K program entry");
    p.prog[e] = KEntry{k.a_src, k.b_src, k.dw, k.dh, k.nchunks, k.a_c0, k.b_k0, k.n_lo, k.n_hi, 0};
    {  // an A source with fewer rows than the output only feeds the leading M tiles (TMA would zero
       // fill the rest: skip those K blocks instead); whole tiles only
      const pcm_asrc& a = d->a[k.a_src];
      const long long rows = d->lin ? a.W : static_cast<long long>(a.B) * d->geoW * d->geoH;
      if (rows < d->M && rows % 128 == 0 && d->ksplit <= 1) {
        p.prog[e].m_hi = static_cast<int>(rows);
        p.filtered = 1;
      }
    }
    nkb += k.nchunks;
    if (k.n_hi != 0) {
      if (k.n_lo % d->block_n != 0 || (k.n_hi % d->block_n != 0 && k.n_hi < d->N) || k.n_hi <= k.n_lo)
        return set_error("pcm_gemm: K entry N range must be aligned to block_n");
      p.filtered = 1;
    }
  }
  p.num_prog = d->num_prog;
  p.lin = d->lin;
  p.M = d->M;
  p.N = d->N;
  p.geoW = d->lin ? 1 : d->geoW;
  p.geoHW = d->lin ? 1 : d->geoW * d->geoH;
  p.block_n = d->block_n;
  p.tiles_m = (d->M + 127) / 128;
  p.tiles_n = (d->N + d->block_n - 1) / d->block_n;
  p.num_kblocks = nkb;
  const int stage_bytes = kATileBytes + d->block_n * 128;
  int S = (kSmemLimit - 1024 - kStagingBytes) / stage_bytes;
  if (S > kMaxStages) S = kMaxStages;
  if (S < 2) return set_error("pcm_gemm: tile too large for shared memory");
  p.num_stages = S;
  p.out = d->out;
  p.bias = d->bias;
  p.rowvec = reinterpret_cast<const bf16*>(d->rowvec);
  p.residual = reinterpret_cast<const bf16*>(d->residual);
  p.osW = d->osW; p.osH = d->osH; p.osB = d->osB;
  p.rowvec_ld = d->rowvec_ld;
  p.epiW = d->epiW > 0 ? d->epiW : 1;
  p.epiHW = d->epiHW > 0 ? d->epiHW : 1;
  p.out_fp32 = d->out_fp32;
  p.round_bf16 = d->round_bf16;
  p.alpha = d->alpha;
  p.act = d->act;
  p.ksplit = 1;
  p.ws = nullptr;
  p.dep_a_map = -1;
  if (d->ksplit > 1 && d->splitk_ws != nullptr && !p.filtered) {
    int ks = d->ksplit;
    if (ks > nkb) ks = nkb;
    const int per = (nkb + ks - 1) / ks;
    ks = (nkb + per - 1) / per;  // every split non-empty
    p.ksplit = ks;
  }

  const size_t smem = static_cast<size_t>(S) * stage_bytes + kStagingBytes + 1024;
  const GemmKernel kernel = gemm_kernel_for(d->block_n);
  static bool attr_set[9] = {};
  if (!attr_set[d->block_n / 32]) {
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
    attr_set[d->block_n / 32] = true;
  }
  if (d->dep_a_src1 > 0 && p.ksplit == 1) {  // (split-K: the finalize kernel follows; keep the plain chain)
    if (d->dep_a_src1 > d->num_a) return set_error("pcm_gemm: bad dep_a_src1");
    p.dep_a_map = d->dep_a_src1 - 1;
  }
  const int tiles = p.tiles_m * p.tiles_n * p.ksplit;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  if (p.ksplit > 1) {
    // pass 1: fp32 partial sums into the workspace; pass 2: epilogue
    GemmParams q = p;
    q.ws = reinterpret_cast<float*>(d->splitk_ws);
    q.bias = nullptr; q.rowvec = nullptr; q.residual = nullptr; q.act = 0;
    CUDA_TRY(launch_pdl(kernel, dim3(grid), dim3(kGemmThreads), smem, stream, q));
    GemmParams f = p;
    f.ws = q.ws;
    f.alpha = 1.f;
    const long long nv = static_cast<long long>(p.M) * ((p.N + 7) / 8);
    int fg = static_cast<int>((nv + 255) / 256);
    if (fg > num_sms() * 8) fg = num_sms() * 8;
    CUDA_TRY(launch_pdl(splitk_finalize_kernel, dim3(fg), dim3(256), 0, stream, f));
    return 0;
  }
  CUDA_TRY(launch_pdl(kernel, dim3(grid), dim3(kGemmThreads), smem, stream, p));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int launch_wgrad(const pcm_wgrad_desc* d, cudaStream_t stream) {
  static WgradParams p;
  memset(&p, 0, sizeof(p));
  if (int rc = encode_asrc(&p.p_map, d->p, d->lin, d->geoW, d->geoH)) return rc;
  if (int rc = encode_asrc(&p.q_map, d->q, d->lin, d->geoW, d->geoH)) return rc;
  if (d->num_taps < 1 || d->num_taps > 9) return set_error("pcm_wgrad: bad tap count");
  p.lin = d->lin;
  p.geoW = d->lin ? 1 : d->geoW;
  p.geoHW = d->lin ? 1 : d->geoW * d->geoH;
  p.M = d->M;
  p.Cp = d->p.C;
  p.q_c0 = d->q_c0;
  p.num_taps = d->num_taps;
  for (int t = 0; t < d->num_taps; ++t) {
    p.dw[t] = d->dw[t];
    p.dh[t] = d->dh[t];
    p.tap_off[t] = d->tap_off[t];
  }
  p.kblocks_total = (d->M + 127) / 128;
  const int ch_tiles = (p.Cp + 127) / 128;
  int ks = d->ksplit;
  if (ks <= 0) {
    // aim for ~2 waves of CTAs, at least 4 token blocks per CTA
    ks = (2 * num_sms() + ch_tiles * d->num_taps - 1) / (ch_tiles * d->num_taps);
    const int max_ks = (p.kblocks_total + 3) / 4;
    if (ks > max_ks) ks = max_ks;
    if (ks < 1) ks = 1;
  }
  if (ks > p.kblocks_total) ks = p.kblocks_total;
  {  // every split non-empty (the deterministic turnstile passes through every blockIdx.z)
    const int per = (p.kblocks_total + ks - 1) / ks;
    ks = (p.kblocks_total + per - 1) / per;
  }
  p.ksplit = ks;
  p.sem = reinterpret_cast<int*>(d->sem);
  p.out = d->out;
  p.os_row = d->os_row;
  p.os_col = d->os_col;
  p.alpha = d->alpha;
  const size_t smem = static_cast<size_t>(kWgStages) * kWgStageBytes + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    CUDA_TRY(cudaFuncSetAttribute(pcm_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  220 * 1024));
    attr_set = true;
  }
  dim3 grid(ch_tiles, d->num_taps, ks);
  CUDA_TRY(launch_pdl(pcm_wgrad_kernel, dim3(grid), dim3(kWgradThreads), smem, stream, p));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace pcm

extern "C" int pcm_gemm(const pcm_gemm_desc* d, void* stream) {
  return pcm::launch_gemm(d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int pcm_wgrad(const pcm_wgrad_desc* d, void* stream) {
  return pcm::launch_wgrad(d, reinterpret_cast<cudaStream_t>(stream));
}
