"""Few-step sampling from a trained PCM LoRA on the CUDA path.

What the reference's validation (train_pcm_lora_sd15.py:120-207, log_validation) runs after training
steps: a StableDiffusionPipeline with DDIMScheduler(timestep_spacing="trailing", clip_sample=False,
set_alpha_to_one=False), the LoRA fused into the UNet (`pipeline.fuse_lora()`), classifier-free guidance
when guidance_scale > 1, eta = 0.  CLIP encoding stays outside: the sampler takes prompt embeddings and
returns the latents the pipeline hands to `vae.decode` (before the 1 / scaling_factor scale), or, given a
pcm_b200.vae.AutoencoderKL, the decoded images (output_type "pt" / "pil").

  * the UNet is an inference copy of the trained network (UNetB200.fused_inference_net): the LoRA targets'
    frozen weights are fused copies W + s B A (pcm_lora_fuse, one launch), every other tensor is shared;
  * each step is n UNet forwards at batch B (or 2B = [uncond; cond] with guidance) and one pcm_sample_step
    launch (CFG mix + DDIM update);
  * on CUDA the whole loop of one shape is captured into a CUDA graph on first use and replayed, with the
    VAE decode and the image postprocessing in the same graph when images are asked for.
"""
import math
import os
import types

import numpy as np
import torch

from . import ops
from .step import sd15_alphas_cumprod

BF16 = torch.bfloat16


def trailing_timesteps(num_inference_steps, num_train_timesteps=1000):
    """DDPMScheduler.set_timesteps with timestep_spacing="trailing" (scheduling_ddpm_modified.py:315-320)."""
    ratio = num_train_timesteps / num_inference_steps
    return np.round(np.arange(num_train_timesteps, 0, -ratio)).astype(np.int64) - 1


def previous_timesteps(timesteps, num_inference_steps, num_train_timesteps=1000):
    """previous_timestep (scheduling_ddpm_modified.py:580-593): t - num_train // n; < 0 on the last step."""
    return timesteps - num_train_timesteps // num_inference_steps


def step_coefficients(alphas_cumprod, num_inference_steps):
    """[(t, sqrt a_t, sqrt(1 - a_t), sqrt a_prev, sqrt(1 - a_prev))] per step, as Python floats (double):
    a = alphas_cumprod[t] (the fp32 table value), a_prev = alphas_cumprod[prev] or alphas_cumprod[0] when
    prev < 0 (set_alpha_to_one=False)."""
    acp = alphas_cumprod.detach().float().cpu()
    n_train = acp.shape[0]
    ts = trailing_timesteps(num_inference_steps, n_train)
    out = []
    for t, tp in zip(ts.tolist(), previous_timesteps(ts, num_inference_steps, n_train).tolist()):
        a = float(acp[t])
        ap = float(acp[tp]) if tp >= 0 else float(acp[0])
        out.append((t, math.sqrt(a), math.sqrt(1.0 - a), math.sqrt(ap), math.sqrt(1.0 - ap)))
    return out


def load_lora_adapter(path):
    """The adapter `save_lora` writes (`adapter_model.safetensors`, peft keys
    `base_model.model.<module>.lora_{A,B}.weight`) as a `<module>.lora_{A,B}.weight` state dict, ready to
    merge into a base UNet state dict for UNetB200.  `path`: the file or its directory."""
    from safetensors.torch import load_file
    f = os.path.join(path, "adapter_model.safetensors") if os.path.isdir(path) else path
    pre = "base_model.model."
    out = {}
    for k, v in load_file(f).items():
        if not k.startswith(pre) or ".lora_" not in k:
            raise ValueError(f"{f}: {k!r} is not a peft LoRA adapter key")
        out[k[len(pre):]] = v
    return out


class PCMSampler:
    """Few-step DDIM ("trailing") sampler over the fused inference copy of a trained UNetB200.

    sampler = PCMSampler(step.unet)
    latents = sampler(prompt_embeds, negative_prompt_embeds, num_inference_steps=4, guidance_scale=7.5,
                      height=512, width=512, generator=torch.Generator("cuda").manual_seed(0))
    sampler.fuse()      # after more training: fuse the current LoRA masters again
    """

    def __init__(self, unet, *, alphas_cumprod=None, prediction_type="epsilon", vae=None):
        """vae: a pcm_b200.vae.AutoencoderKL for output_type "pt" / "pil" (None: latents only)."""
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"Prediction type {prediction_type} currently not supported.")
        self.unet, self.cfg, self.dev, self.vae = unet, unet.cfg, unet.dev, vae
        self.pred_type = 0 if prediction_type == "epsilon" else 1
        acp = sd15_alphas_cumprod() if alphas_cumprod is None else alphas_cumprod
        self.alphas_cumprod = acp.detach().float().cpu()
        self.num_train_timesteps = self.alphas_cumprod.shape[0]
        self.net, self.fuse_table, self.fuse_work = unet.fused_inference_net()
        self._plans = {}
        self._graphs = torch.device(self.dev).type == "cuda"
        self._held = []         # GroupNorm workspaces a captured graph may point at (kept alive)
        self.fuse()

    def fuse(self, master=None):
        """Fuse the LoRA factors of `master` (default: the trained network's fp32 masters; or another flat
        buffer of the same layout, e.g. an EMA copy) into the inference weights: one launch, no copies."""
        master = self.unet.lora_master if master is None else master
        if master.numel() != self.unet.lora_master.numel() or master.dtype != torch.float32:
            raise ValueError("master must be an fp32 buffer of the LoRA master layout")
        ops.lora_fuse(master, self.fuse_table, self.fuse_work, self.unet.scale)

    # ------------------------------------------------------------------------------------------
    def _check(self, prompt_embeds, negative_prompt_embeds, n, guidance_scale, nipp, height, width, latents,
               text_embeds, time_ids, negative_text_embeds):
        cfg = self.cfg
        if not isinstance(n, (int, np.integer)) or isinstance(n, bool) or not 1 <= n <= self.num_train_timesteps:
            raise ValueError(f"num_inference_steps must be an integer in [1, {self.num_train_timesteps}], got {n!r}")
        if not isinstance(nipp, (int, np.integer)) or nipp < 1:
            raise ValueError(f"num_images_per_prompt must be a positive integer, got {nipp!r}")
        if height % 8 != 0 or width % 8 != 0 or height < 8 or width < 8:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        pe = prompt_embeds
        if not torch.is_tensor(pe) or pe.dim() != 3 or pe.shape[2] != cfg.cross_attention_dim:
            raise ValueError(f"prompt_embeds must be [P, S, {cfg.cross_attention_dim}], got "
                             f"{tuple(pe.shape) if torch.is_tensor(pe) else type(pe)}")
        P = pe.shape[0]
        cfg_on = guidance_scale > 1
        if cfg_on:
            if negative_prompt_embeds is None:
                raise ValueError("guidance_scale > 1 needs negative_prompt_embeds")
            if not torch.is_tensor(negative_prompt_embeds) or negative_prompt_embeds.shape != pe.shape:
                raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape, got "
                                 f"{tuple(pe.shape)} and {tuple(getattr(negative_prompt_embeds, 'shape', ()))}")
        B = P * nipp
        h, w = height // 8, width // 8
        if latents is not None and tuple(latents.shape) != (B, cfg.in_channels, h, w):
            raise ValueError(f"latents must be {(B, cfg.in_channels, h, w)}, got {tuple(latents.shape)}")
        if cfg.addition_embed:
            if text_embeds is None or time_ids is None:
                raise ValueError("this UNet needs text_embeds and time_ids (SDXL added conditions)")
            if tuple(text_embeds.shape) != (P, cfg.text_embed_dim):
                raise ValueError(f"text_embeds must be {(P, cfg.text_embed_dim)}, got {tuple(text_embeds.shape)}")
            tid = time_ids.reshape(-1, cfg.num_time_ids) if time_ids.numel() % cfg.num_time_ids == 0 else None
            if tid is None or tid.shape[0] not in (1, P):
                raise ValueError(f"time_ids must be [{cfg.num_time_ids}], [1, {cfg.num_time_ids}] or "
                                 f"[{P}, {cfg.num_time_ids}], got {tuple(time_ids.shape)}")
            if cfg_on:
                if negative_text_embeds is None:
                    raise ValueError("guidance_scale > 1 needs negative_text_embeds (SDXL added conditions)")
                if negative_text_embeds.shape != text_embeds.shape:
                    raise ValueError("`text_embeds` and `negative_text_embeds` must have the same shape")
        elif text_embeds is not None or time_ids is not None or negative_text_embeds is not None:
            raise ValueError("this UNet takes no added conditions (text_embeds / time_ids)")
        return P, B, h, w, cfg_on

    def _plan(self, key):
        plan = self._plans.get(key)
        if plan is not None:
            return plan
        B, h, w, n, cfg_on, S, images = key
        nb = 2 if cfg_on else 1
        dev, cfg = self.dev, self.cfg
        plan = types.SimpleNamespace(B=B, nb=nb, S=S, cfg_on=cfg_on, graph=None)
        # the guidance scale lives in device memory: one captured loop serves every scale > 1
        plan.g = torch.zeros(1, device=dev, dtype=torch.float64) if cfg_on else None
        plan.lat = torch.zeros(nb * B, h, w, cfg.in_channels, device=dev, dtype=torch.float32)
        plan.ctx = torch.zeros(nb * B * S, cfg.cross_attention_dim, device=dev, dtype=BF16)
        plan.added = None
        if cfg.addition_embed:
            plan.added = (torch.zeros(nb * B, cfg.text_embed_dim, device=dev, dtype=BF16),
                          torch.zeros(nb * B, cfg.num_time_ids, device=dev, dtype=torch.int64))
        plan.coef = step_coefficients(self.alphas_cumprod, n)
        plan.ts = torch.tensor([[c[0]] * (nb * B) for c in plan.coef], dtype=torch.int64).to(dev)
        plan.img = plan.u8 = None
        if images:      # [0, 1] NCHW fp32 and uint8 NHWC images of the decoded latents
            plan.img = torch.zeros(B, 3, 8 * h, 8 * w, device=dev, dtype=torch.float32)
            plan.u8 = torch.zeros(B, 8 * h, 8 * w, 3, device=dev, dtype=torch.uint8)
        self._plans[key] = plan
        return plan

    def _run(self, plan):
        """The sampling loop on the plan's static buffers (the sequence a CUDA graph captures)."""
        B = plan.B
        x = plan.lat[:B]
        x2 = plan.lat[B:] if plan.cfg_on else None
        for i, (_, sa, ss, sap, ssp) in enumerate(plan.coef):
            eps = self.net.forward(plan.lat, plan.ts[i], plan.ctx, lora=False, added_cond=plan.added)
            ops.sample_step(eps, x, x, x2, plan.g, sa, ss, sap, ssp, self.pred_type)
        if plan.img is not None:    # the pipeline's vae.decode(latents / scaling_factor) and postprocess
            self.vae.decode_images(x, self.vae.config.scaling_factor, plan.img, plan.u8)

    def _hold_workspaces(self):
        ws = ops._GN_WS.get(torch.device(self.dev))
        if ws is not None and all(ws is not h for h in self._held):
            self._held.append(ws)
        if self.vae is not None:
            self.vae._hold_workspaces()

    def __call__(self, prompt_embeds, negative_prompt_embeds=None, *, num_inference_steps, guidance_scale=1.0,
                 num_images_per_prompt=1, height, width, latents=None, generator=None, text_embeds=None,
                 time_ids=None, negative_text_embeds=None, output_type="latent"):
        """output_type "latent" (default): fp32 NCHW latents [P * num_images_per_prompt, 4, height / 8, width / 8];
        "pt": the decoded fp32 NCHW images in [0, 1] [P * num_images_per_prompt, 3, height, width]; "pil": those
        images as a list of PIL images.  Images of one
        prompt are consecutive (diffusers' `repeat` of the embeddings); with guidance_scale > 1 the UNet runs
        the pipeline's [uncond; cond] batch.  `latents`: the initial noise (default: randn from
        `generator`, init_noise_sigma = 1)."""
        n, g, nipp = num_inference_steps, float(guidance_scale), num_images_per_prompt
        if output_type not in ("latent", "pt", "pil"):
            raise ValueError(f"output_type must be 'latent', 'pt' or 'pil', got {output_type!r}")
        images = output_type != "latent"
        if images and self.vae is None:
            raise ValueError(f"output_type {output_type!r} needs the sampler built with vae=AutoencoderKL(...)")
        P, B, h, w, cfg_on = self._check(prompt_embeds, negative_prompt_embeds, n, g, nipp, height, width,
                                         latents, text_embeds, time_ids, negative_text_embeds)
        cfg = self.cfg
        if latents is None:
            gdev = generator.device if generator is not None else torch.device(self.dev)
            latents = torch.randn(B, cfg.in_channels, h, w, generator=generator, device=gdev, dtype=torch.float32)
        if images:
            self.vae._check_size(height, width, "decode")
        plan = self._plan((B, h, w, int(n), cfg_on, prompt_embeds.shape[1], images))

        def rep(t):
            return t.repeat_interleave(nipp, 0)

        def load():
            if cfg_on:
                plan.g.fill_(g)
            x0 = latents.to(self.dev, torch.float32).permute(0, 2, 3, 1)
            for i in range(plan.nb):
                plan.lat[i * B:(i + 1) * B].copy_(x0)
            halves = [negative_prompt_embeds, prompt_embeds] if cfg_on else [prompt_embeds]
            for i, e in enumerate(halves):
                plan.ctx[i * B * plan.S:(i + 1) * B * plan.S].copy_(rep(e.to(self.dev, BF16)).reshape(B * plan.S, -1))
            if cfg.addition_embed:
                te, tid = plan.added
                pooled = [negative_text_embeds, text_embeds] if cfg_on else [text_embeds]
                tids = time_ids.reshape(-1, cfg.num_time_ids).to(self.dev, torch.int64)
                tids = tids.expand(P, -1) if tids.shape[0] == 1 else tids
                for i, e in enumerate(pooled):
                    te[i * B:(i + 1) * B].copy_(rep(e.to(self.dev, BF16)))
                    tid[i * B:(i + 1) * B].copy_(rep(tids))

        if not self._graphs:
            load()
            self._run(plan)
        else:
            if plan.graph is None:
                self._hold_workspaces()
                load()
                s = torch.cuda.Stream(device=self.dev)
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):          # warm-up: workspaces and modules before the capture
                    self._run(plan)
                torch.cuda.current_stream().wait_stream(s)
                self._hold_workspaces()
                plan.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(plan.graph):
                    self._run(plan)
            load()
            plan.graph.replay()
        if output_type == "pt":
            return plan.img.clone()
        if output_type == "pil":
            from PIL import Image
            return [Image.fromarray(a) for a in plan.u8.cpu().numpy()]
        return plan.lat[:B].permute(0, 3, 1, 2).contiguous()
