/* pcm_b200 -- C ABI of the H100 (sm_90a) PCM-LoRA distillation hot path.
 *
 * The reference (G-U-N/Phased-Consistency-Model) has no FFI/plugin layer: its hot path is Python
 * calling diffusers/peft/torch modules.  This header is the boundary a maintainer binds instead
 * (ctypes stub in INTEGRATION.md).  Every entry point cites the reference call site it replaces
 * (T15 = code/text_to_image_sd15/train_pcm_lora_sd15.py, S15 = scheduling_ddpm_modified.py).
 *
 * Conventions: all pointers are DEVICE pointers owned by the caller (torch tensors); the callee
 * borrows them for the duration of the call; work is enqueued on `stream` (a cudaStream_t passed
 * as void*); return value 0 = ok, negative = error (see pcm_last_error()).  No allocation crosses
 * the ABI.  Activations are NHWC ("channels last") bf16 unless stated otherwise.
 */
#ifndef PCM_B200_H
#define PCM_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCM_MAX_ASRC 6
#define PCM_MAX_BSRC 4
#define PCM_MAX_PROG 24

/* A-operand source: a bf16 NHWC tensor viewed as (C, W, H, B) with element strides. */
typedef struct {
  const void* ptr;
  int32_t C, W, H, B;
  int64_t sW, sH, sB; /* element strides of the W, H, B dims (C is contiguous) */
} pcm_asrc;

/* B-operand source: weights bf16.  kblocked = 0: [N, K] row-major (K contiguous), leading dimension ld.
 * kblocked = 1: K-blocked [K/64][N][64] - the 64-wide K slice of ALL rows is contiguous, so the N x 64
 * operand tile of a K block is one contiguous N*128-byte run in HBM (a row-major tile is N separate
 * 128-byte segments K*2 bytes apart: ~1.2 TB/s measured when small-M layers stream their weights). */
typedef struct {
  const void* ptr;
  int32_t K, N;
  int64_t ld;
  int32_t kblocked;
} pcm_bsrc;

/* One K-program entry: nchunks consecutive 64-wide K blocks read from a[a_src] at channel a_c0..,
 * spatially shifted by (dw, dh) (zero filled outside the image), against b[b_src] columns b_k0...
 * Chunk c multiplies only the K columns both operands have, min(64, a.C - (a_c0 + 64c), b.K - (b_k0 + 64c))
 * rounded up to 16 (TMA zero-fills the operand that ends first): a LoRA entry of rank r (8 <= r <= 256,
 * r % 8 == 0) is ceil(r/64) chunks whose last one is r % 64 wide.  b_k0: a multiple of 64 for a K-blocked
 * B source, of 8 otherwise. */
typedef struct {
  int32_t a_src, b_src, dw, dh, nchunks, a_c0, b_k0;
  uint16_t n_lo, n_hi; /* n_hi > 0: the entry only contributes to output columns [n_lo, n_hi)
                         (multiples of block_n) - lets one launch run several Linear layers that
                         share their input (q/k/v) with per-layer LoRA K blocks */
} pcm_kentry;

/* Implicit-GEMM descriptor: out[m, n] = alpha * sum_k A[m, k] * Bw[n, k] (+bias +rowvec +residual).
 * Replaces nn.Conv2d / nn.Linear (+ peft LoRA branch) calls inside diffusers' UNet2DConditionModel
 * forward/backward issued by T15:1192-1198, 1219-1223, 1238-1244, 1263-1268, 1296. */
typedef struct {
  pcm_asrc a[PCM_MAX_ASRC];
  pcm_bsrc b[PCM_MAX_BSRC];
  pcm_kentry prog[PCM_MAX_PROG];
  int32_t num_a, num_b, num_prog;
  int32_t lin;        /* 1: A sources are plain [M, C] matrices (W = rows), no spatial taps */
  int32_t M, N;       /* output rows (B*H*W tokens) and columns */
  int32_t geoW, geoH; /* conv mode: output image width / height (tile -> TMA coordinates) */
  int32_t block_n;    /* N tile: multiple of 32, <= 256 */
  /* epilogue */
  void* out;          /* bf16 (or fp32 when out_fp32) */
  const float* bias;  /* [N] fp32 or NULL */
  const void* rowvec; /* bf16 [B, rowvec_ld] added per image (time embedding) or NULL */
  const void* residual; /* bf16, same row mapping as out, or NULL */
  int64_t osW, osH, osB; /* element strides of out/residual rows: off = b*osB + h*osH + w*osW */
  int64_t rowvec_ld;
  int32_t epiW, epiHW;   /* row m -> (b = m / epiHW, h = (m % epiHW) / epiW, w = m % epiW) */
  int32_t out_fp32, round_bf16;
  float alpha;
  int32_t act;           /* 0 none, 1 SiLU applied to the result */
  int32_t ksplit;        /* > 1: split the K program over ksplit CTAs per tile (small-M, long-K).  A program
                            with N-ranged entries runs unsplit whatever ksplit says (and then needs no
                            workspace); otherwise ksplit > 1 without splitk_ws is an error */
  void* splitk_ws;       /* fp32 [ksplit, M, N] scratch, 16-byte aligned: one slice of partial sums per K
                            split, added in split order by the finalize kernel */
  int32_t dep_a_src1;    /* 1 + index of the ONLY A source written by the kernel launched immediately
                            before this one on the stream (the layer's LoRA down-projection T), 0 = none.
                            When set, the kernel starts under programmatic dependent launch without
                            waiting for that kernel and only waits right before the first TMA read of
                            this source; M tiles are visited last-to-first so that rows which do not
                            carry the adapter (teacher samples of the merged pass) run while the
                            down-projection is still in flight. Every other input must come from older
                            launches. */
} pcm_gemm_desc;

/* LoRA weight-gradient descriptor: out[ch, r] += alpha * sum_m P[m(+tap), ch] * Q[m, q_c0 + r] for the rank
 * slice r < w = min(64, q.C - q_c0) (a positive multiple of 8); only those w columns of out are stored.  A
 * rank r > 64 takes ceil(r/64) launches (q_c0 + 64j, out advanced by 64j ranks); a slice of a stacked Q
 * narrower than 64 passes a q that ends at the layer's last rank column.
 * Replaces autograd's wgrad of the peft lora_A / lora_B modules (T15:1296). */
typedef struct {
  pcm_asrc p;          /* [tokens, Cp] activation (or grad) */
  pcm_asrc q;          /* [tokens, >= q_c0 + 8] rank-side operand */
  int32_t q_c0;        /* first column of the (at most 64-wide) rank slice of q */
  int32_t lin;
  int32_t M;           /* tokens */
  int32_t geoW, geoH;
  int32_t num_taps;
  int32_t dw[9], dh[9];
  int64_t tap_off[9];  /* element offset into out per tap */
  float* out;          /* fp32, accumulated (see sem) */
  int64_t os_row, os_col; /* out[tap_off + ch*os_row + r*os_col] */
  int32_t ksplit;      /* token-dimension splits (0 = auto) */
  float alpha;
  void* sem;           /* NULL: the token splits accumulate with unordered fp32 atomics.  Otherwise
                          int32[>= ceil(Cp/128) * num_taps], zero-initialised once by the caller: the
                          splits of one output tile then add in split order (bit-reproducible
                          gradients); the kernel leaves the semaphores at zero */
} pcm_wgrad_desc;

const char* pcm_last_error(void);
int pcm_version(void);
int pcm_num_sms(void);

/* wgmma implicit GEMM / conv and LoRA wgrad.  Conv mode takes images whose width divides 128 or is a multiple
 * of 128 (pcm_wgrad: divides 128).  A descriptor the kernels cannot serve is rejected on the
 * host before any CUDA call, pcm_last_error() naming the field: M, N < 1, a null out, conv mode with geoW,
 * geoH, epiW or epiHW < 1, and alignment.  A launch with a bf16 output, no activation and no K split
 * actually run (ksplit <= 1, N-ranged entries, or a program too short to split: ksplit is capped at one
 * split per 64-wide K block) accesses memory 16 bytes at a time: with N >= 32, out, rowvec and bias must
 * be 16-byte aligned and osW, osH, osB and rowvec_ld multiples of 8; with a residual and N >= 8, the
 * residual must be 16-byte aligned and osW, osH, osB multiples of 8 (it is prefetched 8 columns at a
 * time even where the stores are elementwise).  Every other access is elementwise and only needs the
 * pointer aligned to its element.
 * pcm_wgrad: M < 1, a null out, os_row or os_col of zero; out 4-byte aligned, and with os_col == 1 (ranks
 * added in pairs) 8-byte aligned with even os_row and tap_off.
 * pcm_gemm_check / pcm_wgrad_check run exactly those checks and launch nothing.
 * pcm_gemm_plan_rows: the output rows per CTA tile pcm_gemm runs the descriptor with, 128 or 256 (256 for
 * block_n 128 / 160 launches that run unsplit, whose entries without an N or M range hold at least 32 K
 * blocks, whose M-ranged entries end on 256-row boundaries and whose 256-row tiles need at most half the
 * waves of 128-row ones); launches nothing. */
int pcm_gemm(const pcm_gemm_desc* d, void* stream);
int pcm_wgrad(const pcm_wgrad_desc* d, void* stream);
int pcm_gemm_check(const pcm_gemm_desc* d);
int pcm_gemm_plan_rows(const pcm_gemm_desc* d);
int pcm_wgrad_check(const pcm_wgrad_desc* d);

/* ---- GroupNorm(+SiLU) / LayerNorm (NHWC bf16; fp32 statistics) ----------------------------
 * Replace ATen group_norm/layer_norm/silu inside diffusers ResnetBlock2D / Transformer2DModel /
 * BasicTransformerBlock (T15:1192-1198, 1219-1244, 1263-1268) and their backward (T15:1296).
 * x2/C2 (may be NULL/0) is the second half of a channel concat (up-block skip connections).
 * stats: [B, G, 2] (mean, rstd) written by fwd, consumed by bwd; red: [B, G, 2] scratch.
 * ws / ws_bytes: caller-owned scratch of at least pcm_groupnorm_ws_bytes(B, HW, C1 + C2, G) bytes,
 * zero-initialised ONCE (the kernels restore the zeros): per-block partial statistics are merged in
 * block order, so results are bit-reproducible; variance is computed from pivot-shifted sums and
 * Chan's formula (no E[x^2] - mean^2 cancellation). */
int64_t pcm_groupnorm_ws_bytes(int B, int HW, int C, int G);
int pcm_groupnorm_fwd(const void* x1, const void* x2, int C1, int C2, int B, int HW, int G,
                      const float* gamma, const float* beta, float eps, int silu, void* out,
                      float* stats, void* ws, int64_t ws_bytes, void* stream);
/* pcm_groupnorm_fwd over B images, with the per-image block partition of a launch over part_B >= B
 * images: the statistics of image b are merged from the same partials, in the same order, as in that
 * launch, so the outputs are bitwise equal to its rows of images 0..B-1.  Used when the leading images
 * of a batch are normalised again on their own (gradient checkpointing). */
int pcm_groupnorm_fwd_part(const void* x1, const void* x2, int C1, int C2, int B, int part_B, int HW,
                           int G, const float* gamma, const float* beta, float eps, int silu, void* out,
                           float* stats, void* ws, int64_t ws_bytes, void* stream);
int pcm_groupnorm_bwd(const void* dy, const void* x1, const void* x2, int C1, int C2, int B, int HW,
                      int G, const float* gamma, const float* beta, float eps, int silu,
                      const float* stats, float* red, const void* add, void* dx1, void* dx2,
                      float* colsum /* optional fp32 [B, C]: per-image column sums of dx */,
                      void* ws, int64_t ws_bytes, void* stream);
/* stats: [M, 2] (mean, rstd) */
int pcm_layernorm_fwd(const void* x, int M, int C, const float* gamma, const float* beta, float eps,
                      void* out, float* stats, void* stream);
int pcm_layernorm_bwd(const void* dy, const void* x, int M, int C, const float* gamma,
                      const float* stats, const void* add, void* dx, void* stream);

/* ---- attention (flash style; q [B,Sq,H*D], k/v [B,Skv,H*D], row strides ld*) -------------
 * Replaces the xformers / SDPA attention processor enabled at T15:947-961.
 * lse, delta: [B, H, Sq] fp32. */
int pcm_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int H,
                 int Sq, int Skv, int D, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                 float scale, void* stream);
int pcm_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                 const float* lse, float* delta, void* dq, void* dk, void* dv, int B, int H, int Sq,
                 int Skv, int D, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, float scale,
                 void* stream);

/* ---- UNet glue (GEGLU, Upsample2D nearest, 4-channel edge convs, timestep sinusoid, ...) -- */
int pcm_geglu_fwd(const void* u, int64_t M, int F, void* out, void* stream);
int pcm_geglu_bwd(const void* dgg, const void* u, int64_t M, int F, void* du, void* stream);
int pcm_upsample2x_fwd(const void* in, int B, int H, int W, int C, void* out, void* stream);
int pcm_upsample2x_bwd(const void* dout, int B, int H, int W, int C, void* din, void* stream);
/* in: fp32 [B,H,W,4]; w: bf16 [C][3][3][4]; sgn=+1 conv_in forward, -1 conv_out input gradient */
int pcm_conv3x3_c4(const float* in, int B, int H, int W, int C, const void* w, const float* bias,
                   int sgn, int round_in, void* out, void* stream);
int pcm_timestep_embed(const int64_t* t, int B, int C, void* out, void* stream);
int pcm_colsum(const void* x, int B, int HW, int C, void* out, void* stream);
int pcm_add_bf16(const void* a, const void* b, int64_t n, void* out, void* stream);
int pcm_cast_f32_bf16(const float* in, int64_t n, void* out, void* stream);

/* ---- Stable Diffusion VAE (AutoencoderKL) glue around pcm_gemm ---------------------------
 * Replaces, in diffusers' AutoencoderKL (vae.encode(pixels).latent_dist.sample(), T15:1127-1136, and the
 * validation pipeline's vae.decode): the mid-block attention's softmax, DiagonalGaussianDistribution,
 * post_quant_conv and the image postprocessing.
 * pcm_softmax_rows: p[r, :] = bf16(softmax(s[r, :])) with fp32 max and sum, s fp32 [rows, cols] (row stride lds,
 *   16-byte aligned), p bf16 (row stride ldp, 8-byte aligned); cols, lds, ldp multiples of 4.
 * pcm_transpose_bf16: out[b][c][r] = in[b][r][c] for batch bf16 [rows, cols] matrices; ldi / ldo row strides,
 *   bsi / bso batch strides (elements).
 * pcm_latent_dist: quant_conv (1x1, 8 -> 8; w bf16 [8][8], bias fp32 [8]) on h fp32 NHWC [B*HW, 8] (inputs and
 *   result rounded to bf16), then mean = moments[:4], logvar = clamp(moments[4:], -30, 20), std = exp(logvar / 2),
 *   written fp32 NCHW [B, 4, HW].  noise (fp32 NCHW [B, 4, HW]) or NULL: sample = (mean + std * noise) * scale,
 *   each operation rounded on its own.
 * pcm_vae_dec_in: post_quant_conv (1x1, 4 -> 4; w bf16 [4][4], bias fp32 [4]) on bf16(z / div), z fp32 NHWC [M, 4];
 *   out bf16 NHWC [M, 8]: the result in channels 0..3, zeros in 4..7 (the A source of the decoder's conv_in on
 *   pcm_gemm).  z, out 16-byte aligned.
 * pcm_image_exit: v = clamp(x / 2 + 0.5, 0, 1) for x fp32 NHWC [B, HW, C]; out (may be NULL) fp32 NCHW, u8 (may be
 *   NULL) uint8 NHWC round(255 v), round half to even. */
int pcm_softmax_rows(const float* s, int64_t rows, int cols, int64_t lds, void* p, int64_t ldp, void* stream);
int pcm_transpose_bf16(const void* in, int rows, int cols, int64_t ldi, int64_t bsi, int batch, void* out,
                       int64_t ldo, int64_t bso, void* stream);
int pcm_latent_dist(const float* h, int B, int HW, const void* w, const float* bias, const float* noise,
                    float scale, float* mean, float* logvar, float* std, float* sample, void* stream);
int pcm_vae_dec_in(const float* z, int64_t M, const void* w, const float* bias, float div, void* out, void* stream);
int pcm_image_exit(const float* x, int B, int HW, int C, float* out, void* u8, void* stream);

/* ---- PCM solver arithmetic (fused; fp32 latents, batch outermost, `per` elements/sample) ---
 * coef: [B, 16] doubles (internal layout, see csrc/pcm_ops.cu). */
/* T15:1143-1185 + DDIMSolver tables T15:289-303 + phase start T15:321-341 + c_skip T15:250-259 */
int pcm_prepare(const float* alphas_cumprod, int num_train, int num_ddim, const int64_t* inf_idx,
                int multiphase, const int64_t* index, const float* w, int B, int bf16_mode,
                double* coef, int64_t* start_t, int64_t* t, int64_t* end_t, void* stream);
/* DDPMScheduler.add_noise, S15:500-524 (T15:1178) */
int pcm_add_noise(const float* x, const float* noise, const double* coef, int64_t per, int B,
                  int bf16_mode, float* out, void* stream);
/* predicted_origin x2 + CFG mix + DDIMSolver.ddim_step, T15:1224-1258.
 * pred_type: 0 = epsilon, 1 = v_prediction (predicted_origin, T15:268-280) */
int pcm_teacher_step(const float* eps_c, const float* eps_u, const float* noisy, const double* coef,
                     int64_t per, int B, int pred_type, float* x_prev, void* stream);
/* Opt-in multi-substep teacher solve (num_substeps > 1; the reference does ONE step, T15:1217-1258):
 * one DDIM sub-step t_cur[b] -> t_next[b] (t_next < 0 = the solver's alpha_cumprods[0] entry) of the
 * CFG-mixed prediction; with a single sub-step it equals pcm_teacher_step bit for bit */
int pcm_teacher_substep(const float* eps_c, const float* eps_u, const float* x_cur,
                        const float* alphas_cumprod, const int64_t* t_cur, const int64_t* t_next,
                        const double* coef, int64_t per, int B, int pred_type, float* x_next, void* stream);
/* T15:1200-1212 + 1269-1293: loss (0 = huber, 1 = l2), d loss / d eps_student, optional dumps */
int pcm_loss(const float* eps_s, const float* eps_t, const float* noisy, const float* x_prev,
             const double* coef, int64_t per, int B, int loss_type, float huber_c, int pred_type,
             float* loss_out, float* d_eps, float* model_pred, float* target, void* stream);
/* DDPMScheduler.noise_travel, S15:526-554 */
int pcm_noise_travel(const float* x, const float* noise, const float* alphas_cumprod,
                     const int64_t* t_cur, const int64_t* t_tgt, int64_t per, int B, float* out,
                     void* stream);

/* out = ca[b]*x + cb[b]*y in float64: DDIMSolver.ddim_step / ddim_style_multiphase_pred
 * (T15:313-341) for callers that use the solver object directly */
int pcm_axpby_f64(const float* x, const float* y, const double* ca, const double* cb, int64_t per,
                  int B, double* out, void* stream);

/* Flow-matching (SD3) steps, fp32 in the reference's operation order (bit-identical to its torch ops):
 * mode 0 = PCMFMDeterministicScheduler.step (pcm_fm_deterministic_scheduler.py:226-233),
 * mode 1 = PCMFMStochasticScheduler.step (pcm_fm_stochastic_scheduler.py:226-233, z = noise),
 * mode 2 = scale_noise (pcm_fm_deterministic_scheduler.py:90-115).  sig / sig_next: one value per sample.
 * (EulerSolver.euler_step / euler_style_multiphase_pred, train_pcm_lora_sd3.py:160-226, return float64
 * like the reference and go through pcm_axpby_f64.) */
int pcm_fm_step(const float* x, const float* v, const float* z, const float* sig, const float* sig_next,
                int64_t per, int B, int mode, float* out, void* stream);

/* ---- optimiser on the flat fp32 LoRA buffer (T15:1297-1301) ------------------------------- */
/* out: PCM_SUMSQ_WS_DOUBLES doubles, zero-initialised once: out[0] = sum of squares; the rest is
 * scratch (block counter + per-block partials added in block order: bit-reproducible norm) */
#define PCM_SUMSQ_WS_DOUBLES 1024
int pcm_grad_sumsq(const float* g, int64_t n, double* out, void* stream);
/* state: device float[2] = {lr, step}; step is incremented on device before the update */
int pcm_adamw_clip(float* p, float* g, float* m, float* v, int64_t n, float* state, float beta1,
                   float beta2, float eps, float weight_decay, float max_norm, float inv_world,
                   const double* sumsq, int zero_grad, void* stream);
/* update_ema(target_params, source_params, rate), T15:344-355 (defined but never called by the
 * reference loop; offered as the opt-in EMA target): targ = rate*targ + (1-rate)*src */
int pcm_ema_update(float* targ, const float* src, int64_t n, float rate, void* stream);
/* table: num_entries x 9 int64 {a_off, b_off, a_fwd, sb_fwd, sb_t, a_t, cin|taps<<32, n|r<<32,
 * work_begin}; writes bf16 operand copies A, s*B, (s*B)^T, A^T.  Work = min(r, 64) x 64 tiles: per entry
 * ceil(r/64) * (taps*cin/64 + n/64), work_begin its prefix sum, total_work the sum */
int pcm_lora_refresh(const float* master, const void* table, int num_entries, int64_t total_work,
                     float scale, void* opnd, void* stream);
/* LoRA fused into the frozen weights for inference (peft fuse_lora), out of place on the K-blocked
 * [K/64][N_total][64] bf16 operands: dst[n0+n, k] = bf16(float(src[n0+n, k]) + scale * sum_r B[n,r] A[r,k]),
 * fp32 sum in ascending rank order, one rounding.  table: num_entries x 8 int64 {a_off, b_off (fp32
 * master elements; A [r][K], B [n][r]), src, dst (device addresses of the stacked operands),
 * n0 | N_total<<32, K | r<<32, n, work_begin}; n and K multiples of 64, 8 <= r <= 256, r % 8 == 0.
 * Work = 64 x 64 tiles: per entry (n/64) * (K/64), work_begin its prefix sum, total_work the sum */
int pcm_lora_fuse(const float* master, const void* table, int num_entries, int64_t total_work, float scale,
                  void* stream);
/* One eta = 0 DDIM step of the few-step sampler (DDIMScheduler trailing, set_alpha_to_one=False) after
 * the pipeline's CFG mix.  cfg != 0 (guidance scale > 1): eps holds 2B samples [uncond; cond] and is
 * mixed eps_u + g (eps_c - eps_u) with g = *guidance (device double); cfg == 0: B samples, guidance unread.  pred_type 0 = epsilon, 1 = v_prediction.
 * x_out = sqrt(a_prev) x0 + sqrt(1-a_prev) eps in double, rounded to fp32; x_out2 (may be NULL) gets the
 * same values.  x_out may alias x. */
int pcm_sample_step(const float* eps, const float* x, float* x_out, float* x_out2, int64_t per, int B,
                    int cfg, const double* guidance, double sqrt_a_t, double sqrt_1m_a_t, double sqrt_a_prev,
                    double sqrt_1m_a_prev, int pred_type, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PCM_B200_H */
