"""CPU oracle of the few-step sampler (test infrastructure only): the reference validation pipeline's loop
(train_pcm_lora_sd15.py:120-207: StableDiffusionPipeline + DDIMScheduler(timestep_spacing="trailing",
clip_sample=False, set_alpha_to_one=False) after `fuse_lora()`, eta = 0) over oracle/unet_ref.py with the
merged weights W + s B A.  Timesteps and previous timesteps follow DDPMScheduler.set_timesteps /
previous_timestep (scheduling_ddpm_modified.py:315-320, 580-593), pinned by tests/golden/sampler_math.pt."""
import numpy as np
import torch


def merge_lora(cfg, params, emulate_bf16=False):
    """peft fuse_lora on the oracle's parameter dict: W + s (B A) for every LoRA target, adapters dropped
    (emulate_bf16: the frozen W is the bf16 weight the CUDA path holds)."""
    s = cfg.lora_alpha / cfg.lora_rank
    out = {k: v for k, v in params.items() if ".lora_" not in k}
    for k in params:
        if not k.endswith(".lora_A.weight"):
            continue
        name = k[:-len(".lora_A.weight")]
        W = params[name + ".weight"].float()
        if emulate_bf16:
            W = W.to(torch.bfloat16).float()
        A = params[k].double().reshape(cfg.lora_rank, -1)
        Bm = params[name + ".lora_B.weight"].double().reshape(W.shape[0], cfg.lora_rank)
        out[name + ".weight"] = W + (s * (Bm @ A)).float().reshape(W.shape)
    return out


def sample_ref(cfg, params, prompt_embeds, negative_prompt_embeds=None, *, num_inference_steps, latents,
               guidance_scale=1.0, alphas_cumprod=None, prediction_type="epsilon", added_cond=None,
               negative_added_cond=None, emulate_bf16=False):
    """latents: NCHW initial noise [B, 4, h, w]; prompt_embeds [B, S, D] (one row per image);
    added_cond / negative_added_cond: SDXL dict(text_embeds [B, *], time_ids [B, 6]).  Returns the final
    latents (fp32 NCHW).  The DDIM update runs in float64 from the fp32 alpha table."""
    from oracle import pcm_ref, unet_ref
    acp = pcm_ref.sd15_alphas_cumprod() if alphas_cumprod is None else alphas_cumprod
    n_train = acp.shape[0]
    net = unet_ref.UNetRef(cfg, merge_lora(cfg, params, emulate_bf16), use_lora=False, emulate_bf16=emulate_bf16)
    n = num_inference_steps
    ts = np.round(np.arange(n_train, 0, -n_train / n)).astype(np.int64) - 1
    x = latents.float()
    B = x.shape[0]
    g = float(guidance_scale)
    for t in ts.tolist():
        tp = t - n_train // n
        a = float(acp[t])
        ap = float(acp[tp]) if tp >= 0 else float(acp[0])
        if g > 1:
            addc = None
            if added_cond is not None:
                addc = {k: torch.cat([negative_added_cond[k], added_cond[k]]) for k in added_cond}
            e2 = net(torch.cat([x, x]), torch.full((2 * B,), t, dtype=torch.int64),
                     torch.cat([negative_prompt_embeds, prompt_embeds]), addc).double()
            e = e2[:B] + g * (e2[B:] - e2[:B])
        else:
            e = net(x, torch.full((B,), t, dtype=torch.int64), prompt_embeds, added_cond).double()
        xd = x.double()
        if prediction_type == "epsilon":
            x0, pe = (xd - (1 - a) ** 0.5 * e) / a ** 0.5, e
        else:
            x0, pe = a ** 0.5 * xd - (1 - a) ** 0.5 * e, a ** 0.5 * e + (1 - a) ** 0.5 * xd
        x = (ap ** 0.5 * x0 + (1 - ap) ** 0.5 * pe).float()
    return x
