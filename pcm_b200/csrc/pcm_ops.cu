// Fused PCM solver arithmetic: the ~100 tiny ATen launches of the reference loop
// (train_pcm_lora_sd15.py:1139-1293) collapsed into four kernels.
//
//   pcm_prepare      : T15:1143-1185  timestep / phase bookkeeping, add_noise (S15:500-524),
//                      per-sample coefficient table (alpha/sigma gathers, DDIM tables of
//                      DDIMSolver.__init__ T15:289-303, phase start of
//                      ddim_style_multiphase_pred T15:321-341, c_skip/c_out T15:250-259)
//   pcm_teacher_step : T15:1224-1258  predicted_origin x2, CFG mix, DDIMSolver.ddim_step
//   pcm_loss         : T15:1200-1212 + 1269-1293  student/target x0 recovery, phase jump,
//                      boundary mix, Huber / L2 loss, and the loss gradient w.r.t. the student
//                      epsilon (the seed of the UNet backward, T15:1296)
//   pcm_noise_travel : S15:526-554 (adversarial variant re-noising)
// Latent tensors are fp32, any layout with the batch dimension outermost (per = elements/sample).
// Solver coefficients are evaluated in double like the reference's float64 DDIM tables.
#include "common.cuh"
#include "host_common.h"
#include "../../include/pcm_b200.h"

namespace pcm {

// coefficient table, per sample (doubles)
enum {
  kAlphaS = 0,  // sqrt(acp[start_t])        (fp32 table value)
  kSigmaS,      // sqrt(1-acp[start_t])
  kAlphaT,      // sqrt(acp[t])
  kSigmaT,      // sqrt(1-acp[t])
  kAp,          // sqrt(acp_prev[phase start])     (double)
  kSp,          // sqrt(1-acp_prev[phase start])
  kAi,          // sqrt(acp_prev[index])
  kSi,          // sqrt(1-acp_prev[index])
  kCskip,       // 1 if index is a phase start
  kW,           // guidance scale
  kNoiseA,      // add_noise coefficients (possibly bf16-rounded like the reference under autocast)
  kNoiseS,
  kCoefN = 16
};

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__global__ void pcm_prepare_kernel(const float* __restrict__ acp, int num_train, int num_ddim,
                                   const long long* __restrict__ inf_idx, int multiphase,
                                   const long long* __restrict__ index, const float* __restrict__ w,
                                   int B, int bf16_mode, double* __restrict__ coef,
                                   long long* __restrict__ start_t, long long* __restrict__ t_out,
                                   long long* __restrict__ end_t) {
  griddep_sync();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int ratio = num_train / num_ddim;  // DDIMSolver.step_ratio (T15:291)
  const long long idx = index[b];
  const long long st = (idx + 1) * ratio - 1;  // ddim_timesteps[idx]            (T15:292-294)
  long long tt = st - ratio;                   // T15:1152
  if (tt < 0) tt = 0;                          // T15:1153-1155
  // phase start: largest inference index <= idx (T15:329-335)
  long long p = inf_idx[0];
  int is_start = 0;
  for (int j = 0; j < multiphase; ++j) {
    if (inf_idx[j] <= idx) p = inf_idx[j];
    if (inf_idx[j] == idx) is_start = 1;       // torch.isin (T15:251)
  }
  // ddim_alpha_cumprods_prev[i] = acp[0] if i == 0 else acp[i*ratio - 1]   (T15:297-299)
  const double ap = static_cast<double>(p == 0 ? acp[0] : acp[p * ratio - 1]);
  const double ai = static_cast<double>(idx == 0 ? acp[0] : acp[idx * ratio - 1]);
  double* c = coef + static_cast<long long>(b) * kCoefN;
  c[kAlphaS] = static_cast<double>(sqrtf(acp[st]));        // alpha_schedule (T15:808)
  c[kSigmaS] = static_cast<double>(sqrtf(1.f - acp[st]));  // sigma_schedule (T15:809)
  c[kAlphaT] = static_cast<double>(sqrtf(acp[tt]));
  c[kSigmaT] = static_cast<double>(sqrtf(1.f - acp[tt]));
  c[kAp] = sqrt(ap);
  c[kSp] = sqrt(1.0 - ap);
  c[kAi] = sqrt(ai);
  c[kSi] = sqrt(1.0 - ai);
  c[kCskip] = is_start ? 1.0 : 0.0;
  float wv = w[b];
  float na, ns;
  if (bf16_mode) {
    // add_noise casts alphas_cumprod to the sample dtype first (S15:510) and w is cast to
    // latents.dtype (T15:1185)
    const float a16 = rbf(acp[st]);
    na = rbf(sqrtf(a16));
    ns = rbf(sqrtf(rbf(1.f - a16)));
    wv = rbf(wv);
  } else {
    na = sqrtf(acp[st]);
    ns = sqrtf(1.f - acp[st]);
  }
  c[kW] = static_cast<double>(wv);
  c[kNoiseA] = static_cast<double>(na);
  c[kNoiseS] = static_cast<double>(ns);
  start_t[b] = st;
  t_out[b] = tt;
  end_t[b] = (p == 0) ? 0 : p * ratio - 1;  // ddim_timesteps_prev[p] (T15:296, 341)
}

__global__ void pcm_add_noise_kernel(const float* __restrict__ x, const float* __restrict__ noise,
                                     const double* __restrict__ coef, long long per,
                                     long long total, int bf16_mode, float* __restrict__ out) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const double* c = coef + (i / per) * kCoefN;
    float xv = x[i], nv = noise[i];
    if (bf16_mode) {
      xv = rbf(xv);
      nv = rbf(nv);
    }
    float y;
    if (bf16_mode) {
      // the reference evaluates add_noise on bf16 tensors: every op rounds (S15:513-523)
      y = rbf(rbf(static_cast<float>(c[kNoiseA]) * xv) + rbf(static_cast<float>(c[kNoiseS]) * nv));
    } else {
      y = static_cast<float>(c[kNoiseA]) * xv + static_cast<float>(c[kNoiseS]) * nv;
    }
    out[i] = y;
  }
}

__global__ void pcm_teacher_step_kernel(const float* __restrict__ eps_c,
                                        const float* __restrict__ eps_u,
                                        const float* __restrict__ noisy,
                                        const double* __restrict__ coef, long long per,
                                        long long total, int pred_type,
                                        float* __restrict__ x_prev) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const double* c = coef + (i / per) * kCoefN;
    const float al = static_cast<float>(c[kAlphaS]), sg = static_cast<float>(c[kSigmaS]);
    const float w = static_cast<float>(c[kW]);
    const float ec = eps_c[i], eu = eps_u[i], xn = noisy[i];
    // predicted_origin: epsilon (T15:272) or v_prediction (T15:275)
    const float x0c = pred_type == 0 ? (xn - sg * ec) / al : al * xn - sg * ec;
    const float x0u = pred_type == 0 ? (xn - sg * eu) / al : al * xn - sg * eu;
    const float px0 = x0c + w * (x0c - x0u);  // T15:1254
    const float pe = ec + w * (ec - eu);      // T15:1255-1257
    const double xp = c[kAi] * static_cast<double>(px0) + c[kSi] * static_cast<double>(pe);
    x_prev[i] = static_cast<float>(xp);       // consumed as x_prev.float() (T15:1264)
  }
}

// single block: deterministic reduction
__global__ void pcm_loss_kernel(const float* __restrict__ eps_s, const float* __restrict__ eps_t,
                                const float* __restrict__ noisy, const float* __restrict__ x_prev,
                                const double* __restrict__ coef, long long per, long long total,
                                int loss_type, float huber_c, int pred_type,
                                float* __restrict__ loss_out, float* __restrict__ d_eps,
                                float* __restrict__ model_pred_out,
                                float* __restrict__ target_out) {
  griddep_sync();
  __shared__ double s_part[32];
  double acc = 0.0;
  const double inv_n = 1.0 / static_cast<double>(total);
  for (long long i = threadIdx.x; i < total; i += blockDim.x) {
    const double* c = coef + (i / per) * kCoefN;
    const float es = eps_s[i], et = eps_t[i], xn = noisy[i], xp = x_prev[i];
    // student: x0 = (noisy - sigma*eps)/alpha (T15:1200-1207); jump to the phase start (T15:1209);
    // c_skip_start = 0, c_out_start = 1 (T15:256-259, 1212)
    const float als = static_cast<float>(c[kAlphaS]), sgs = static_cast<float>(c[kSigmaS]);
    const float alt = static_cast<float>(c[kAlphaT]), sgt = static_cast<float>(c[kSigmaT]);
    const float x0s = pred_type == 0 ? (xn - sgs * es) / als : als * xn - sgs * es;
    const double mp = c[kAp] * static_cast<double>(x0s) + c[kSp] * static_cast<double>(es);
    // target: same network at (x_prev, t) (T15:1263-1279), then c_skip/c_out mix (T15:1280)
    const float x0t = pred_type == 0 ? (xp - sgt * et) / alt : alt * xp - sgt * et;
    const double tj = c[kAp] * static_cast<double>(x0t) + c[kSp] * static_cast<double>(et);
    const double tg = c[kCskip] * static_cast<double>(xp) + (1.0 - c[kCskip]) * tj;
    const float mpf = static_cast<float>(mp), tgf = static_cast<float>(tg);  // .float() T15:1285,1290
    const float d = mpf - tgf;
    float l, dl;
    if (loss_type == 0) {  // huber (T15:1287-1293)
      const float r = sqrtf(d * d + huber_c * huber_c);
      l = r - huber_c;
      dl = d / r;
    } else {  // l2 (T15:1283-1286)
      l = d * d;
      dl = 2.f * d;
    }
    acc += static_cast<double>(l);
    // d model_pred / d eps_s = Sp - Ap * sigma / alpha  (v_prediction: Sp - Ap * sigma)
    const double dmp = pred_type == 0 ? c[kSp] - c[kAp] * c[kSigmaS] / c[kAlphaS]
                                      : c[kSp] - c[kAp] * c[kSigmaS];
    if (d_eps) d_eps[i] = static_cast<float>(static_cast<double>(dl) * inv_n * dmp);
    if (model_pred_out) model_pred_out[i] = mpf;
    if (target_out) target_out[i] = tgf;
  }
  // block reduce
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < (blockDim.x >> 5) ? s_part[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) loss_out[0] = static_cast<float>(v * inv_n);
  }
}

// noise_travel (S15:526-554): x' = sqrt(a_tgt/a_cur) x + sqrt(1 - a_tgt/a_cur) noise
__global__ void pcm_noise_travel_kernel(const float* __restrict__ x, const float* __restrict__ noise,
                                        const float* __restrict__ acp,
                                        const long long* __restrict__ t_cur,
                                        const long long* __restrict__ t_tgt, long long per,
                                        long long total, float* __restrict__ out) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / per;
    const float r = acp[t_tgt[b]] / acp[t_cur[b]];
    out[i] = sqrtf(r) * x[i] + sqrtf(1.f - r) * noise[i];
  }
}

// out[i] = ca[b] * x[i] + cb[b] * y[i] in double (DDIMSolver.ddim_step / multiphase jump, which
// return float64 tensors in the reference because its alpha table is float64, T15:297-303)
__global__ void pcm_axpby_f64_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                     const double* __restrict__ ca, const double* __restrict__ cb,
                                     long long per, long long total, double* __restrict__ out) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / per;
    out[i] = ca[b] * static_cast<double>(x[i]) + cb[b] * static_cast<double>(y[i]);
  }
}

static inline int grid_for(long long total) {
  long long g = (total + 255) / 256;
  if (g > num_sms() * 8) g = num_sms() * 8;
  return static_cast<int>(g < 1 ? 1 : g);
}

}  // namespace pcm

using namespace pcm;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int pcm_prepare(const float* acp, int num_train, int num_ddim, const int64_t* inf_idx,
                           int multiphase, const int64_t* index, const float* w, int B,
                           int bf16_mode, double* coef, int64_t* start_t, int64_t* t,
                           int64_t* end_t, void* stream) {
  CUDA_TRY(launch_pdl(pcm_prepare_kernel, dim3((B + 63) / 64), dim3(64), 0, ST(stream), acp, num_train, num_ddim, reinterpret_cast<const long long*>(inf_idx), multiphase,
      reinterpret_cast<const long long*>(index), w, B, bf16_mode, coef,
      reinterpret_cast<long long*>(start_t), reinterpret_cast<long long*>(t),
      reinterpret_cast<long long*>(end_t)));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
extern "C" int pcm_add_noise(const float* x, const float* noise, const double* coef, int64_t per,
                             int B, int bf16_mode, float* out, void* stream) {
  const long long total = per * B;
  CUDA_TRY(launch_pdl(pcm_add_noise_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), x, noise, coef, per, total,
                                                                bf16_mode, out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
extern "C" int pcm_teacher_step(const float* eps_c, const float* eps_u, const float* noisy,
                                const double* coef, int64_t per, int B, int pred_type,
                                float* x_prev, void* stream) {
  const long long total = per * B;
  if (pred_type != 0 && pred_type != 1) return set_error("pcm_teacher_step: bad prediction type");
  CUDA_TRY(launch_pdl(pcm_teacher_step_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), eps_c, eps_u, noisy, coef, per,
                                                                   total, pred_type, x_prev));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
extern "C" int pcm_loss(const float* eps_s, const float* eps_t, const float* noisy,
                        const float* x_prev, const double* coef, int64_t per, int B, int loss_type,
                        float huber_c, int pred_type, float* loss_out, float* d_eps,
                        float* model_pred, float* target, void* stream) {
  const long long total = per * B;
  if (pred_type != 0 && pred_type != 1) return set_error("pcm_loss: bad prediction type");
  CUDA_TRY(launch_pdl(pcm_loss_kernel, dim3(1), dim3(1024), 0, ST(stream), eps_s, eps_t, noisy, x_prev, coef, per, total,
                                              loss_type, huber_c, pred_type, loss_out, d_eps,
                                              model_pred, target));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
extern "C" int pcm_noise_travel(const float* x, const float* noise, const float* acp,
                                const int64_t* t_cur, const int64_t* t_tgt, int64_t per, int B,
                                float* out, void* stream) {
  const long long total = per * B;
  CUDA_TRY(launch_pdl(pcm_noise_travel_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), x, noise, acp, reinterpret_cast<const long long*>(t_cur),
      reinterpret_cast<const long long*>(t_tgt), per, total, out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_axpby_f64(const float* x, const float* y, const double* ca, const double* cb,
                             int64_t per, int B, double* out, void* stream) {
  const long long total = per * B;
  CUDA_TRY(launch_pdl(pcm_axpby_f64_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), x, y, ca, cb, per, total, out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Flow-matching (SD3) solver / scheduler steps: train_pcm_lora_sd3.py:160-226 (EulerSolver) and
// pcm_fm_{deterministic,stochastic}_scheduler.py (step, scale_noise).  One fused elementwise kernel,
// fp32 arithmetic in the reference's operation order WITHOUT fma contraction, so results are
// bit-identical to the reference's torch elementwise ops.
//   mode 0  deterministic step (FMD:226-233): denoised = x - v*s; d = (x - denoised)/s;
//                                             out = x + d*(s_next - s)
//   mode 1  stochastic step   (FMS:226-233): denoised = x - v*s; out = (1 - s_next)*denoised + s_next*z
//   mode 2  scale_noise       (FMD:90-115):  out = s*z + (1 - s)*x
// s / s_next: one value per sample (sig[b], sig_next[b]); z = noise (modes 1, 2).
// ------------------------------------------------------------------------------------------
namespace pcm {
__global__ void pcm_fm_step_kernel(const float* __restrict__ x, const float* __restrict__ v,
                                   const float* __restrict__ z, const float* __restrict__ sig,
                                   const float* __restrict__ sig_next, long long per, long long total,
                                   int mode, float* __restrict__ out) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / per;
    const float s = sig[b];
    const float xv = x[i];
    float o;
    if (mode == 0) {
      const float den = __fsub_rn(xv, __fmul_rn(v[i], s));
      const float d = __fdiv_rn(__fsub_rn(xv, den), s);
      o = __fadd_rn(xv, __fmul_rn(d, __fsub_rn(sig_next[b], s)));
    } else if (mode == 1) {
      const float den = __fsub_rn(xv, __fmul_rn(v[i], s));
      const float sn = sig_next[b];
      o = __fadd_rn(__fmul_rn(__fsub_rn(1.f, sn), den), __fmul_rn(sn, z[i]));
    } else {
      o = __fadd_rn(__fmul_rn(s, z[i]), __fmul_rn(__fsub_rn(1.f, s), xv));
    }
    out[i] = o;
  }
}
}  // namespace pcm

extern "C" int pcm_fm_step(const float* x, const float* v, const float* z, const float* sig,
                           const float* sig_next, int64_t per, int B, int mode, float* out,
                           void* stream) {
  if (mode < 0 || mode > 2) return set_error("pcm_fm_step: bad mode");
  const long long total = per * B;
  CUDA_TRY(launch_pdl(pcm_fm_step_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), x, v, z, sig, sig_next,
                      static_cast<long long>(per), total, mode, out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Opt-in multi-substep teacher solve: one DDIM sub-step of the CFG-mixed teacher prediction from
// train timestep t_cur[b] to t_next[b] (the reference takes the whole DDIM interval in ONE step,
// T15:1217-1258; with num_substeps = 1 this kernel reproduces pcm_teacher_step bit for bit).
// alpha / sigma at t_cur are the fp32 schedule values (alpha_schedule / sigma_schedule, T15:808-809);
// the target point uses acp[t_next] in double like DDIMSolver.ddim_alpha_cumprods_prev
// (t_next < 0 -> acp[0], the solver's convention for its first entry, T15:297-299).
// ------------------------------------------------------------------------------------------
namespace pcm {
__global__ void pcm_teacher_substep_kernel(const float* __restrict__ eps_c, const float* __restrict__ eps_u,
                                           const float* __restrict__ x_cur, const float* __restrict__ acp,
                                           const long long* __restrict__ t_cur,
                                           const long long* __restrict__ t_next,
                                           const double* __restrict__ coef, long long per, long long total,
                                           int pred_type, float* __restrict__ x_next) {
  griddep_sync();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / per;
    const float a_cur = acp[t_cur[b]];
    const float al = sqrtf(a_cur), sg = sqrtf(1.f - a_cur);
    const long long tn = t_next[b];
    const double an = static_cast<double>(tn < 0 ? acp[0] : acp[tn]);
    const float w = static_cast<float>(coef[b * kCoefN + kW]);
    const float ec = eps_c[i], eu = eps_u[i], xn = x_cur[i];
    const float x0c = pred_type == 0 ? (xn - sg * ec) / al : al * xn - sg * ec;
    const float x0u = pred_type == 0 ? (xn - sg * eu) / al : al * xn - sg * eu;
    const float px0 = x0c + w * (x0c - x0u);
    const float pe = ec + w * (ec - eu);
    x_next[i] = static_cast<float>(sqrt(an) * static_cast<double>(px0) + sqrt(1.0 - an) * static_cast<double>(pe));
  }
}
}  // namespace pcm

// ------------------------------------------------------------------------------------------
// One step of the few-step sampler (the reference's validation pipeline: StableDiffusionPipeline with
// DDIMScheduler(timestep_spacing="trailing", set_alpha_to_one=False), eta = 0, T15:120-207):
//   cfg:          eps = eps_u + g (eps_c - eps_u) on the [uncond; cond] batch of 2B samples, g = *guidance
//                 (device memory, so one captured loop serves every guidance scale > 1)
//   epsilon:      x0 = (x - sqrt(1-a_t) eps) / sqrt(a_t)
//   v_prediction: x0 = sqrt(a_t) x - sqrt(1-a_t) v,  eps = sqrt(a_t) v + sqrt(1-a_t) x
//   x_prev = sqrt(a_prev) x0 + sqrt(1-a_prev) eps
// The four square roots are host doubles; the arithmetic runs in double with one rounding to fp32.
// x_out2 (optional) receives a second copy: the other half of the next step's 2B-sample UNet input.
// ------------------------------------------------------------------------------------------
namespace pcm {
__global__ void pcm_sample_step_kernel(const float* __restrict__ eps, const float* x,
                                       float* x_out, float* x_out2, long long total, int cfg,
                                       const double* __restrict__ guidance, double sa, double ss, double sap,
                                       double ssp, int pred_type) {
  griddep_sync();
  const double g = cfg ? *guidance : 1.0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    double e;
    if (cfg) {
      const double eu = eps[i], ec = eps[total + i];
      e = eu + g * (ec - eu);
    } else {
      e = eps[i];
    }
    const double xv = x[i];
    double x0, pe;
    if (pred_type == 0) {
      x0 = (xv - ss * e) / sa;
      pe = e;
    } else {
      x0 = sa * xv - ss * e;
      pe = sa * e + ss * xv;
    }
    const float o = static_cast<float>(sap * x0 + ssp * pe);
    x_out[i] = o;
    if (x_out2) x_out2[i] = o;
  }
}
}  // namespace pcm

extern "C" int pcm_sample_step(const float* eps, const float* x, float* x_out, float* x_out2, int64_t per,
                               int B, int cfg, const double* guidance, double sqrt_a_t, double sqrt_1m_a_t,
                               double sqrt_a_prev, double sqrt_1m_a_prev, int pred_type, void* stream) {
  if (pred_type != 0 && pred_type != 1) return set_error("pcm_sample_step: bad prediction type");
  if (cfg && !guidance) return set_error("pcm_sample_step: guidance needs its device scalar");
  const long long total = per * B;
  CUDA_TRY(launch_pdl(pcm_sample_step_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), eps, x, x_out,
                      x_out2, total, cfg ? 1 : 0, guidance, sqrt_a_t, sqrt_1m_a_t, sqrt_a_prev,
                      sqrt_1m_a_prev, pred_type));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int pcm_teacher_substep(const float* eps_c, const float* eps_u, const float* x_cur,
                                   const float* alphas_cumprod, const int64_t* t_cur,
                                   const int64_t* t_next, const double* coef, int64_t per, int B,
                                   int pred_type, float* x_next, void* stream) {
  const long long total = per * B;
  if (pred_type != 0 && pred_type != 1) return set_error("pcm_teacher_substep: bad prediction type");
  CUDA_TRY(launch_pdl(pcm_teacher_substep_kernel, dim3(grid_for(total)), dim3(256), 0, ST(stream), eps_c, eps_u,
                      x_cur, alphas_cumprod, reinterpret_cast<const long long*>(t_cur),
                      reinterpret_cast<const long long*>(t_next), coef, static_cast<long long>(per), total,
                      pred_type, x_next));
  CUDA_TRY(cudaGetLastError());
  return 0;
}
