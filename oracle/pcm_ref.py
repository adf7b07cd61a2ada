"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the PCM distillation math of the reference,
code/text_to_image_sd15/train_pcm_lora_sd15.py (T15) and
scheduling_ddpm_modified.py (S15).  Every function cites the lines it follows.  The restatement
is PINNED against the reference's own functions executed verbatim (AST-extracted from the
read-only tree by tests/golden/make_golden.py -> tests/golden/pcm_math.pt; checked by
tests/test_oracle.py).  The UNet inside the step is oracle/unet_ref.py (parity unpinned: the
reference delegates it to diffusers/peft which are not installed here).
"""
import numpy as np
import torch

from .unet_ref import UNetRef, lora_keys


def sd15_alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    """DDPMScheduler `scaled_linear` schedule (S15:211-215; SD1.5 scheduler config T15:805-807)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def append_dims(x, target_dims):  # T15:240-247
    if target_dims - x.ndim < 0:
        raise ValueError(f"input has {x.ndim} dims but target_dims is {target_dims}, which is less")
    return x[(...,) + (None,) * (target_dims - x.ndim)]


def scalings_for_boundary_conditions_target(index, selected_indices):  # T15:250-253
    c_skip = torch.isin(index, selected_indices).float()
    return c_skip, 1.0 - c_skip


def scalings_for_boundary_conditions_online(index, selected_indices):  # T15:256-259
    return torch.zeros_like(index).float(), torch.ones_like(index).float()


def extract_into_tensor(a, t, x_shape):  # T15:283-286
    b = t.shape[0]
    return a.gather(-1, t).reshape(b, *((1,) * (len(x_shape) - 1)))


def predicted_origin(model_output, timesteps, sample, prediction_type, alphas, sigmas):  # T15:268-280
    s = extract_into_tensor(sigmas, timesteps, sample.shape)
    a = extract_into_tensor(alphas, timesteps, sample.shape)
    if prediction_type == "epsilon":
        return (sample - s * model_output) / a
    if prediction_type == "v_prediction":
        return a * sample - s * model_output
    raise ValueError(f"Prediction type {prediction_type} currently not supported.")


def inference_indices(num_ddim, multiphase):  # T15:322-325 == T15:1157-1160
    return np.floor(np.linspace(0, num_ddim, num=multiphase, endpoint=False)).astype(np.int64)


class DDIMSolverRef:
    """T15:289-341.  Note ddim_alpha_cumprods_prev is float64 (built from a Python list)."""

    def __init__(self, alpha_cumprods, timesteps=1000, ddim_timesteps=50):
        self.step_ratio = timesteps // ddim_timesteps
        ts = (np.arange(1, ddim_timesteps + 1) * self.step_ratio).round().astype(np.int64) - 1
        self.ddim_alpha_cumprods = torch.from_numpy(alpha_cumprods[ts])
        self.ddim_timesteps_prev = torch.from_numpy(np.asarray([0] + ts[:-1].tolist())).long()
        self.ddim_alpha_cumprods_prev = torch.from_numpy(
            np.asarray([alpha_cumprods[0]] + alpha_cumprods[ts[:-1]].tolist()))
        self.ddim_timesteps = torch.from_numpy(ts).long()

    def ddim_step(self, pred_x0, pred_noise, timestep_index):  # T15:313-319
        a = extract_into_tensor(self.ddim_alpha_cumprods_prev, timestep_index, pred_x0.shape)
        return a.sqrt() * pred_x0 + (1.0 - a).sqrt() * pred_noise

    def ddim_style_multiphase_pred(self, pred_x0, pred_noise, timestep_index, multiphase):  # T15:321-341
        inf = torch.from_numpy(inference_indices(len(self.ddim_timesteps), multiphase)).long()
        # largest phase-start index <= timestep_index  (expand / >= / flip / argmax in the reference)
        pos = (timestep_index[:, None] >= inf[None, :]).long().sum(1) - 1
        p = inf[pos]
        a = extract_into_tensor(self.ddim_alpha_cumprods_prev, p, pred_x0.shape)
        return a.sqrt() * pred_x0 + (1.0 - a).sqrt() * pred_noise, self.ddim_timesteps_prev[p]


def add_noise(alphas_cumprod, x, noise, timesteps):  # S15:500-524 (stock DDPMScheduler.add_noise)
    ac = alphas_cumprod.to(dtype=x.dtype)
    sa = (ac[timesteps] ** 0.5).flatten()
    so = ((1 - ac[timesteps]) ** 0.5).flatten()
    while len(sa.shape) < len(x.shape):
        sa, so = sa.unsqueeze(-1), so.unsqueeze(-1)
    return sa * x + so * noise


def noise_travel(alphas_cumprod, x, noise, t_cur, t_tgt):  # S15:526-554
    ac = alphas_cumprod.to(dtype=x.dtype)
    a_cur, a_tgt = ac[t_cur], ac[t_tgt]
    ratio = (a_tgt / a_cur)
    sa = (ratio ** 0.5).flatten()
    so = ((1 - ratio) ** 0.5).flatten()
    while len(sa.shape) < len(x.shape):
        sa, so = sa.unsqueeze(-1), so.unsqueeze(-1)
    return sa * x + so * noise


def pcm_step_ref(cfg, params, batch, *, multiphase, num_ddim=50, loss_type="huber", huber_c=1e-3,
                 prediction_type="epsilon", apply_cfg_solver=True, emulate_bf16=False,
                 need_grad=True, round_eps_bf16=None, teacher_substeps=1):
    """One iteration of the reference loop, T15:1139-1293, on explicit inputs.

    batch: latents [B,4,H,W], noise, index [B] int64, w [B], prompt_embeds [B,77,D],
           uncond_prompt_embeds [B,77,D]  (all fp32 CPU tensors)
    Returns dict(loss, grads{name: tensor}, model_pred, target, x_prev, eps_student, ...).
    The target network is the SAME LoRA student under no_grad (T15:1261-1268; update_ema is never
    called in the reference)."""
    ac = sd15_alphas_cumprod()
    alpha_schedule, sigma_schedule = torch.sqrt(ac), torch.sqrt(1 - ac)      # T15:808-809
    solver = DDIMSolverRef(ac.numpy(), 1000, num_ddim)                        # T15:811-815
    if round_eps_bf16 is None:
        round_eps_bf16 = emulate_bf16
    P = dict(params)
    lk = lora_keys(P)
    if need_grad:
        for k in lk:
            P[k] = P[k].detach().clone().requires_grad_(True)
    student = UNetRef(cfg, P, use_lora=True, emulate_bf16=emulate_bf16)
    teacher = UNetRef(cfg, P, use_lora=False, emulate_bf16=emulate_bf16)

    def rq(x):  # dtype of tensors the reference keeps in weight_dtype (bf16 under mixed precision)
        return x.to(torch.bfloat16).float() if emulate_bf16 else x

    latents, noise = rq(batch["latents"]), rq(batch["noise"])                 # T15:1136, 1139
    index, w = batch["index"], batch["w"]
    prompt, uncond = batch["prompt_embeds"], batch["uncond_prompt_embeds"]
    # SDXL (train_pcm_lora_sdxl_adv.py:1094-1133, 1215-1221): added_cond_kwargs; the unconditional
    # teacher pass uses ZERO pooled text embeddings and the same time ids
    addc = addu = None
    if "text_embeds" in batch:
        addc = dict(text_embeds=rq(batch["text_embeds"]), time_ids=batch["time_ids"])
        addu = dict(text_embeds=torch.zeros_like(batch["text_embeds"]), time_ids=batch["time_ids"])
    topk = 1000 // num_ddim                                                   # T15:1143-1146
    start_t = solver.ddim_timesteps[index]                                    # T15:1151
    t = torch.clamp(start_t - topk, min=0)                                    # T15:1152-1155
    inf = torch.from_numpy(inference_indices(num_ddim, multiphase)).long()    # T15:1157-1163
    c_skip_s, c_out_s = [append_dims(x, 4) for x in scalings_for_boundary_conditions_online(index, inf)]
    c_skip, c_out = [append_dims(x, 4) for x in scalings_for_boundary_conditions_target(index, inf)]
    if emulate_bf16:   # latents are weight_dtype (bf16) tensors in the reference: run its exact op sequence
        noisy = add_noise(ac, latents.bfloat16(), noise.bfloat16(), start_t).float()
    else:
        noisy = add_noise(ac, latents, noise, start_t)                        # T15:1178
    w4 = rq(w.reshape(-1, 1, 1, 1))                                           # T15:1183-1185

    eps = student(noisy, start_t, prompt, addc)                               # T15:1192-1198
    x0 = predicted_origin(eps, start_t, noisy, prediction_type, alpha_schedule, sigma_schedule)
    model_pred, end_t = solver.ddim_style_multiphase_pred(x0, eps, index, multiphase)  # T15:1209
    model_pred = c_skip_s * noisy + c_out_s * model_pred                      # T15:1212

    with torch.no_grad():                                                     # T15:1217-1258
        eps_c = teacher(noisy, start_t, prompt, addc)
        x0_c = predicted_origin(eps_c, start_t, noisy, prediction_type, alpha_schedule, sigma_schedule)
        if apply_cfg_solver:
            eps_u = teacher(noisy, start_t, uncond, addu)
            x0_u = predicted_origin(eps_u, start_t, noisy, prediction_type, alpha_schedule, sigma_schedule)
        else:
            eps_u, x0_u = eps_c, x0_c
        pred_x0 = x0_c + w4 * (x0_c - x0_u)                                   # T15:1254
        pred_noise = eps_c + w4 * (eps_c - eps_u)                             # T15:1255-1257
        if teacher_substeps == 1:
            x_prev = solver.ddim_step(pred_x0, pred_noise, index)             # T15:1258 (float64)
        else:
            # opt-in extension (not in the reference): k DDIM sub-steps over the same interval
            k, dt = teacher_substeps, topk // teacher_substeps
            acd = ac.double()
            x_cur, t_cur = noisy, start_t
            for j in range(k):
                t_next = start_t - (j + 1) * dt
                a_n = torch.where(t_next < 0, acd[0], acd[t_next.clamp(min=0)]).reshape(-1, 1, 1, 1)
                x_next = a_n.sqrt() * pred_x0 + (1.0 - a_n).sqrt() * pred_noise
                if j == k - 1:
                    x_prev = x_next
                    break
                x_cur, t_cur = x_next.float(), t_next.clamp(min=0)
                e_c = teacher(x_cur, t_cur, prompt, addc)
                e_u = teacher(x_cur, t_cur, uncond, addu) if apply_cfg_solver else e_c
                p_c = predicted_origin(e_c, t_cur, x_cur, prediction_type, alpha_schedule, sigma_schedule)
                p_u = predicted_origin(e_u, t_cur, x_cur, prediction_type, alpha_schedule, sigma_schedule)
                pred_x0 = p_c + w4 * (p_c - p_u)
                pred_noise = e_c + w4 * (e_c - e_u)

        eps_t = student(x_prev.float(), t, prompt, addc)                      # T15:1263-1268
        x0_t = predicted_origin(eps_t, t, x_prev, prediction_type, alpha_schedule, sigma_schedule)
        target, end_t2 = solver.ddim_style_multiphase_pred(x0_t, eps_t, index, multiphase)
        target = c_skip * x_prev + c_out * target                             # T15:1280

    if loss_type == "l2":                                                     # T15:1283-1293
        loss = torch.nn.functional.mse_loss(model_pred.float(), target.float(), reduction="mean")
    else:
        loss = torch.mean(torch.sqrt((model_pred.float() - target.float()) ** 2 + huber_c ** 2) - huber_c)
    out = dict(loss=loss.detach(), model_pred=model_pred.detach(), target=target.detach(),
               x_prev=x_prev.detach(), eps_student=eps.detach(), eps_cond=eps_c, eps_uncond=eps_u,
               eps_target=eps_t, noisy=noisy, start_timesteps=start_t, timesteps=t, end_timesteps=end_t)
    if need_grad:
        loss.backward()                                                       # T15:1296
        out["grads"] = {k: P[k].grad.detach() for k in lk}
    return out


def clip_and_adamw_ref(params, grads, state, *, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                       max_grad_norm=1.0, world=1):
    """T15:1297-1301: clip_grad_norm_(max_norm) over all LoRA grads, then torch.optim.AdamW.step."""
    keys = sorted(grads)
    total = torch.sqrt(sum((grads[k].double() ** 2).sum() for k in keys)).float()
    coef = torch.clamp(max_grad_norm / (total + 1e-6), max=1.0) if max_grad_norm > 0 else torch.tensor(1.0)
    state["step"] = state.get("step", 0) + 1
    s = state["step"]
    for k in keys:
        g = grads[k] * coef
        m = state.setdefault("m." + k, torch.zeros_like(g))
        v = state.setdefault("v." + k, torch.zeros_like(g))
        p = params[k]
        p.mul_(1 - lr * weight_decay)
        m.mul_(betas[0]).add_(g, alpha=1 - betas[0])
        v.mul_(betas[1]).addcmul_(g, g, value=1 - betas[1])
        denom = (v.sqrt() / (1 - betas[1] ** s) ** 0.5).add_(eps)
        p.addcdiv_(m, denom, value=-lr / (1 - betas[0] ** s))
    return total


def make_batch(cfg, B, hw, seed=0, num_ddim=50, w_min=4.0, w_max=5.0, index=None, zero_uncond=False):
    """Synthetic inputs of SURVEY.md section 8(d): CPU generator, fixed seeds per tensor."""
    def g(s):
        return torch.Generator().manual_seed(seed * 1000 + s)
    latents = torch.randn(B, 4, hw, hw, generator=g(0))
    noise = torch.randn(B, 4, hw, hw, generator=g(1))
    prompt = torch.randn(B, 77, cfg.cross_attention_dim, generator=g(2))
    uncond = torch.randn(1, 77, cfg.cross_attention_dim, generator=g(3)).repeat(B, 1, 1)
    if index is None:
        index = torch.randint(0, num_ddim, (B,), generator=g(4))
    w = (w_max - w_min) * torch.rand(B, generator=g(5)) + w_min
    out = dict(latents=latents, noise=noise, prompt_embeds=prompt, uncond_prompt_embeds=uncond,
               index=index.long(), w=w)
    if getattr(cfg, "addition_embed", False):   # SDXL: pooled text embedding + (orig size, crop, target size)
        out["text_embeds"] = torch.randn(B, cfg.text_embed_dim, generator=g(6))
        res = float(hw * 8)
        out["time_ids"] = torch.tensor([[res, res, 0.0, 0.0, res, res]] * B).long()
        if zero_uncond:
            out["uncond_prompt_embeds"] = torch.zeros_like(uncond)          # TXL:1215-1218
    return out
