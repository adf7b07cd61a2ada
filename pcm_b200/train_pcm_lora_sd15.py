#!/usr/bin/env python
"""`train_pcm_lora_sd15` entry point on the CUDA path.

Keeps the reference script's command line (flag names / defaults of
code/text_to_image_sd15/train_pcm_lora_sd15.py:381-735) so existing launch recipes
(`train_pcm_lora_sd15.sh`) keep working; the per-iteration hot path runs through libpcm_b200.so
(PCMTrainStep).  What is NOT here (out of scope, SURVEY.md section 8): the image dataset, VAE and CLIP
encoders, validation image logging, hub upload.  Inputs to the step are therefore either
  --synthetic            seeded random latents / text embeddings (benchmark + parity mode), or
  --latent_cache DIR     *.pt files holding {"latents" [B,4,h,w], "prompt_embeds" [B,77,768]}
                         produced upstream by the reference's own VAE/CLIP preprocessing, plus the CLIP
                         encoding of the empty prompt (T15:1053-1059) either per file
                         ("uncond_prompt_embeds" [B or 1,77,768]) or once via --uncond_embeds FILE.
Checkpoints `checkpoint-N/` hold the LoRA adapter AND the optimiser state (AdamW moments, step, lr,
host RNG), rotate under --checkpoints_total_limit and resume with --resume_from_checkpoint
(accelerator.save_state / load_state semantics, T15:1080-1105, 1308-1343).
Launch: `python -m pcm_b200.train_pcm_lora_sd15 ...` or
`python -m torch.distributed.run --nproc-per-node N -m pcm_b200.train_pcm_lora_sd15 ...`.
"""
import argparse
import glob
import json
import math
import os
import shutil
import sys
import time

import torch

from . import config, dp, lr_schedules, weights
from .step import PCMTrainStep


def parse_args(argv=None, extra=None):
    p = argparse.ArgumentParser(description="PCM-LoRA distillation on H100")
    if extra is not None:
        extra(p)
    # ---- flags of the reference script, verbatim names / defaults ----
    p.add_argument("--pretrained_teacher_model", type=str, default=None,
                   help="directory with unet/diffusion_pytorch_model.safetensors; omitted -> seeded random init")
    p.add_argument("--pretrained_vae_model_name_or_path", type=str, default=None)
    p.add_argument("--teacher_revision", type=str, default=None)
    p.add_argument("--revision", type=str, default=None)
    p.add_argument("--output_dir", type=str, default="lcm-xl-distilled")
    p.add_argument("--cache_dir", type=str, default=None)
    p.add_argument("--seed", type=int, default=None)
    p.add_argument("--logging_dir", type=str, default="logs")
    p.add_argument("--report_to", type=str, default="tensorboard")
    p.add_argument("--checkpointing_steps", type=int, default=500)
    p.add_argument("--checkpoints_total_limit", type=int, default=None)
    p.add_argument("--resume_from_checkpoint", type=str, default=None)
    p.add_argument("--resolution", type=int, default=512)
    p.add_argument("--center_crop", default=False, action="store_true")
    p.add_argument("--random_flip", action="store_true")
    p.add_argument("--dataloader_num_workers", type=int, default=8)
    p.add_argument("--train_batch_size", type=int, default=16)
    p.add_argument("--num_train_epochs", type=int, default=100)
    p.add_argument("--max_train_steps", type=int, default=None)
    p.add_argument("--max_train_samples", type=int, default=None)
    p.add_argument("--learning_rate", type=float, default=1e-4)
    p.add_argument("--scale_lr", action="store_true", default=False)
    p.add_argument("--lr_scheduler", type=str, default="constant")
    p.add_argument("--lr_warmup_steps", type=int, default=500)
    p.add_argument("--gradient_accumulation_steps", type=int, default=1)
    p.add_argument("--use_8bit_adam", action="store_true")
    p.add_argument("--adam_beta1", type=float, default=0.9)
    p.add_argument("--adam_beta2", type=float, default=0.999)
    p.add_argument("--adam_weight_decay", type=float, default=1e-2)
    p.add_argument("--adam_epsilon", type=float, default=1e-08)
    p.add_argument("--max_grad_norm", default=1.0, type=float)
    p.add_argument("--proportion_empty_prompts", type=float, default=0)
    p.add_argument("--w_min", type=float, default=5.0)
    p.add_argument("--w_max", type=float, default=15.0)
    p.add_argument("--num_ddim_timesteps", type=int, default=50)
    p.add_argument("--loss_type", type=str, default="l2", choices=["l2", "huber"])
    p.add_argument("--huber_c", type=float, default=0.001)
    p.add_argument("--lora_rank", type=int, default=64)
    p.add_argument("--mixed_precision", type=str, default=None, choices=["no", "fp16", "bf16"])
    p.add_argument("--allow_tf32", action="store_true")
    p.add_argument("--cast_teacher_unet", action="store_true")
    p.add_argument("--enable_xformers_memory_efficient_attention", action="store_true")
    p.add_argument("--gradient_checkpointing", action="store_true")
    p.add_argument("--local_rank", type=int, default=-1)
    p.add_argument("--validation_steps", type=int, default=200)
    p.add_argument("--push_to_hub", action="store_true")
    p.add_argument("--hub_token", type=str, default=None)
    p.add_argument("--hub_model_id", type=str, default=None)
    p.add_argument("--tracker_project_name", type=str, default="text2image-fine-tune")
    p.add_argument("--not_apply_cfg_solver", action="store_true")
    p.add_argument("--multiphase", default=8, type=int)
    # ---- additions of this implementation ----
    p.add_argument("--synthetic", action="store_true", help="seeded synthetic latents / text embeddings")
    p.add_argument("--latent_cache", type=str, default=None)
    p.add_argument("--uncond_embeds", type=str, default=None,
                   help=".pt tensor [1 or B,77,768]: CLIP encoding of the empty prompt (T15:1053-1059)")
    p.add_argument("--no_cuda_graph", action="store_true")
    p.add_argument("--log_every", type=int, default=10)
    p.add_argument("--prediction_type", type=str, default="epsilon", choices=["epsilon", "v_prediction"],
                   help="noise_scheduler.config.prediction_type of the teacher (T15:1204, 1228)")
    p.add_argument("--ema_decay", type=float, default=None,
                   help="opt-in EMA target (update_ema, T15:344-355); default: target = student like the reference")
    p.add_argument("--validation_prompt_embeds", type=str, default=None,
                   help=".pt dict {prompt_embeds [P,77,D]} (+ text_embeds [P,*], time_ids [P or 1,6] for SDXL): "
                        "sample 4 images per prompt in --multiphase steps every --validation_steps (T15:1345-1365) "
                        "into output_dir/validation/step-N/cfg-{g}.pt")
    args = p.parse_args(argv)
    env_local_rank = int(os.environ.get("LOCAL_RANK", -1))   # same override as the reference
    if env_local_rank != -1 and env_local_rank != args.local_rank:
        args.local_rank = env_local_rank
    if args.proportion_empty_prompts < 0 or args.proportion_empty_prompts > 1:
        raise ValueError("`--proportion_empty_prompts` must be in the range [0, 1].")
    if args.gradient_accumulation_steps != 1:
        raise ValueError("pcm_b200 runs one optimiser step per iteration (all reference recipes use 1)")
    if args.use_8bit_adam:
        raise ValueError("--use_8bit_adam (bitsandbytes) is not provided: an 80 GB H100 holds the fp32 AdamW state of the LoRA factors (0.54 GB)")
    if args.mixed_precision == "no":
        raise ValueError("--mixed_precision no (fp32 compute) is not provided: the CUDA path computes with "
                         "bf16 operands and fp32 accumulation; use bf16")
    if args.mixed_precision == "fp16":
        # every shipped recipe passes fp16 (train_pcm_lora_sd15.sh:9).  fp16 and bf16 run on the same
        # tensor-core rate; this implementation stores activations as bf16 (8 exponent bits: no
        # GradScaler / overflow skipping needed) - documented deviation, DESIGN.md section 4.
        print("pcm_b200: --mixed_precision fp16 runs the bf16 path (same rate, wider range, no loss scaling)",
              file=sys.stderr)
    config.check_lora_rank(args.lora_rank)        # peft takes any r; the kernels take 8 <= r <= 256, r % 8 == 0
    if args.lr_scheduler not in lr_schedules.SCHEDULES:
        raise ValueError(f"{args.lr_scheduler} is not a valid SchedulerType, please select one of "
                         f"{list(lr_schedules.SCHEDULES)}.")
    return args


def _lr_at(args, step, world=1):
    """Learning rate of optimiser step `step` (0-based): diffusers get_scheduler(...) as stepped by
    accelerate (T15:1026-1031, 1300)."""
    return lr_schedules.lr_at(args.lr_scheduler, args.learning_rate, step, args.lr_warmup_steps,
                              args.max_train_steps, num_processes=world)


def find_resume_path(output_dir, resume_from_checkpoint):
    """T15:1082-1090: explicit path -> its basename; "latest" -> highest checkpoint-N in output_dir."""
    if resume_from_checkpoint != "latest":
        return os.path.basename(resume_from_checkpoint)
    if not os.path.isdir(output_dir):
        return None
    dirs = [d for d in os.listdir(output_dir) if d.startswith("checkpoint")]
    dirs = sorted(dirs, key=lambda x: int(x.split("-")[1]))
    return dirs[-1] if len(dirs) > 0 else None


def rotate_checkpoints(output_dir, total_limit):
    """T15:1311-1337: before saving, keep at most `total_limit - 1` existing checkpoints."""
    if total_limit is None:
        return
    ckpts = [d for d in os.listdir(output_dir) if d.startswith("checkpoint")]
    ckpts = sorted(ckpts, key=lambda x: int(x.split("-")[1]))
    if len(ckpts) >= total_limit:
        for d in ckpts[0:len(ckpts) - total_limit + 1]:
            shutil.rmtree(os.path.join(output_dir, d))


def save_state(st, cfg, path, global_step, gen):
    """accelerator.save_state (T15:1339-1341): adapter weights + optimiser state + RNG."""
    save_lora(st, cfg, path)
    sd = st.state_dict()
    sd.update(global_step=global_step, rng_state=gen.get_state(), lora_rank=cfg.lora_rank)
    torch.save(sd, os.path.join(path, "pcm_b200_state.pt"))


def load_state(st, path, gen):
    """accelerator.load_state (T15:1099-1100)."""
    f = os.path.join(path, "pcm_b200_state.pt")
    if not os.path.exists(f):
        raise FileNotFoundError(f"{f} not found: checkpoints written before optimiser state was saved cannot be resumed")
    sd = torch.load(f)
    if sd.get("lora_rank", st.unet.r) != st.unet.r:
        raise ValueError(f"{path} holds a rank-{sd['lora_rank']} LoRA adapter; this run trains rank {st.unet.r} "
                         f"(--lora_rank must match the checkpoint to resume from it)")
    st.load_state_dict(sd)
    gen.set_state(sd["rng_state"])
    return int(sd["global_step"])


def validation_enabled(args):
    """Validation sampling is opt-in: it runs only with --validation_prompt_embeds."""
    return args.validation_prompt_embeds is not None


def validation_guidances(config_sdxl):
    """log_validation's guidance scales: 1 and 7.5 for SD1.5 (T15:1345-1365), 1 for SDXL (TXL:1578)."""
    return (1.0,) if config_sdxl else (1.0, 7.5)


class _Validation:
    """log_validation (T15:120-207) on latents: the LoRA fused into an inference copy of the UNet, each
    prompt sampled 4 times in `multiphase` DDIM-trailing steps from one generator seeded with --seed, at every
    guidance scale; latents and seed saved to output_dir/validation/step-N/cfg-{g}.pt."""

    def __init__(self, args, st, cfg, uncond):
        d = torch.load(args.validation_prompt_embeds)
        self.pe = d["prompt_embeds"].float().reshape(-1, 77, cfg.cross_attention_dim)
        P = self.pe.shape[0]
        self.ne = None if uncond is None else uncond.float().reshape(-1, 77, cfg.cross_attention_dim)[:1].repeat(P, 1, 1)
        self.extra = {}
        if cfg.addition_embed:
            te = d["text_embeds"].float()
            self.extra = dict(text_embeds=te, time_ids=d["time_ids"].long().reshape(-1, cfg.num_time_ids),
                              negative_text_embeds=torch.zeros_like(te))
        self.args, self.st, self.cfg = args, st, cfg
        self.guidances = validation_guidances(cfg.addition_embed)
        if any(g > 1 for g in self.guidances) and self.ne is None:
            raise SystemExit("validation with guidance > 1 needs the empty-prompt embedding (--uncond_embeds)")
        self.sampler = None

    def __call__(self, global_step):
        from .sampling import PCMSampler
        if self.sampler is None:
            self.sampler = PCMSampler(self.st.unet, alphas_cumprod=self.st.acp, prediction_type=self.args.prediction_type)
        else:
            self.sampler.fuse()
        out_dir = os.path.join(self.args.output_dir, "validation", f"step-{global_step}")
        os.makedirs(out_dir, exist_ok=True)
        seed, res = self.args.seed, self.args.resolution
        dev = self.st.unet.dev
        for g in self.guidances:
            gen = None if seed is None else torch.Generator(device=dev).manual_seed(seed)
            lats = []
            for i in range(self.pe.shape[0]):        # one pipeline call per prompt (T15:163-175)
                ex = {}
                if self.extra:
                    tid = self.extra["time_ids"]
                    ex = dict(text_embeds=self.extra["text_embeds"][i:i + 1],
                              time_ids=tid[i:i + 1] if tid.shape[0] > 1 else tid,
                              negative_text_embeds=self.extra["negative_text_embeds"][i:i + 1])
                lats.append(self.sampler(self.pe[i:i + 1], None if self.ne is None else self.ne[i:i + 1],
                                         num_inference_steps=self.args.multiphase, guidance_scale=g,
                                         num_images_per_prompt=4, height=res, width=res, generator=gen, **ex))
            torch.save({"latents": torch.cat(lats).cpu(), "seed": seed, "guidance_scale": g},
                       os.path.join(out_dir, f"cfg-{g}.pt"))


def main(args):
    rank, world, _ = dp.env_rank_world()
    local = max(args.local_rank, 0)
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    pg = None
    if world > 1:
        pg = dp.init_process_group("nccl", dev)
    if args.seed is not None:
        torch.manual_seed(dp.rank_seed(args.seed, rank))        # set_seed(args.seed + process_index)
    import dataclasses
    cfg = getattr(args, "_cfg", None) or dataclasses.replace(getattr(args, "_base_cfg", config.SD15),
                                                               lora_rank=args.lora_rank)
    if args.pretrained_teacher_model:
        from safetensors.torch import load_file
        sd = load_file(os.path.join(args.pretrained_teacher_model, "unet", "diffusion_pytorch_model.safetensors"))
        sd.update({k: v for k, v in weights.synthetic_state_dict(cfg, args.seed or 0, lora_b_std=0.0).items()
                   if ".lora_" in k})              # peft init: A kaiming-uniform, B zeros
    else:
        sd = weights.synthetic_state_dict(cfg, args.seed or 0)
    hw = args.resolution // 8
    B = args.train_batch_size
    # --scale_lr is declared by the reference (T15:535-540) but never read: it has no effect there either
    st = PCMTrainStep(cfg, sd, dev, batch=B, height=hw, width=hw, multiphase=args.multiphase,
                      num_ddim_timesteps=args.num_ddim_timesteps, loss_type=args.loss_type,
                      huber_c=args.huber_c, lr=args.learning_rate, betas=(args.adam_beta1, args.adam_beta2),
                      adam_eps=args.adam_epsilon, weight_decay=args.adam_weight_decay,
                      max_grad_norm=args.max_grad_norm, apply_cfg_solver=not args.not_apply_cfg_solver,
                      process_group=pg, prediction_type=args.prediction_type, ema_decay=args.ema_decay,
                      gradient_checkpointing=args.gradient_checkpointing)
    del sd
    files = sorted(glob.glob(os.path.join(args.latent_cache, "*.pt"))) if args.latent_cache else []
    if not files and not args.synthetic:
        raise SystemExit("need --synthetic or --latent_cache (the image/VAE/CLIP pipeline is out of scope)")
    gen = torch.Generator().manual_seed(dp.rank_seed(args.seed or 0, rank))
    uncond = None
    if args.uncond_embeds:
        uncond = torch.load(args.uncond_embeds).float().reshape(-1, 77, cfg.cross_attention_dim)
    elif cfg.addition_embed:
        # SDXL: zero unconditional embeddings (train_pcm_lora_sdxl_adv.py:1215-1221)
        uncond = torch.zeros(1, 77, cfg.cross_attention_dim)
    elif args.synthetic:
        # synthetic stand-in for text_encoder([""] * B): one embedding repeated over the batch
        uncond = torch.randn(1, 77, cfg.cross_attention_dim, generator=torch.Generator().manual_seed(3))

    # T15:1018-1024: steps per epoch = len(dataloader); max_train_steps defaults to epochs * that
    if files:
        steps_per_epoch = max(1, math.ceil(len(files) / world))
    elif args.max_train_samples:
        steps_per_epoch = max(1, math.ceil(args.max_train_samples / (B * world)))
    else:
        steps_per_epoch = None
    if args.max_train_steps is None:
        if steps_per_epoch is None:
            raise SystemExit("--synthetic needs --max_train_steps (or --max_train_samples for an epoch length)")
        args.max_train_steps = args.num_train_epochs * steps_per_epoch

    def next_batch(i):
        extra = ()
        if files:
            d = torch.load(files[(i * world + rank) % len(files)])
            lat, pe = d["latents"].float(), d["prompt_embeds"].float()
            unc = d.get("uncond_prompt_embeds", uncond)
            if unc is None:
                raise SystemExit(
                    "the CFG-augmented solver needs the CLIP encoding of the empty prompt (T15:1053-1059, "
                    "1237-1258): put `uncond_prompt_embeds` into the cache files or pass --uncond_embeds")
            unc = unc.float().reshape(-1, 77, cfg.cross_attention_dim)
            if cfg.addition_embed:
                extra = (d["text_embeds"].bfloat16(), d["time_ids"].long())
        else:
            lat = torch.randn(B, 4, hw, hw, generator=gen)
            pe = torch.randn(B, 77, cfg.cross_attention_dim, generator=gen)
            unc = uncond
            if cfg.addition_embed:   # pooled text embedding + (original size, crop top-left, target size)
                res = args.resolution
                extra = (torch.randn(B, cfg.text_embed_dim, generator=gen).bfloat16(),
                         torch.tensor([[res, res, 0, 0, res, res]] * B))
        if unc.shape[0] == 1:
            unc = unc.repeat(B, 1, 1)
        noise = torch.randn(B, 4, hw, hw, generator=gen)
        index = torch.randint(0, args.num_ddim_timesteps, (B,), generator=gen)
        w = (args.w_max - args.w_min) * torch.rand(B, generator=gen) + args.w_min
        nhwc = lambda x: x.permute(0, 2, 3, 1).contiguous()
        return (nhwc(lat), nhwc(noise), index, w, pe.bfloat16(), unc.bfloat16()) + tuple(extra)

    os.makedirs(args.output_dir, exist_ok=True)
    global_step = 0
    if args.resume_from_checkpoint:                # T15:1080-1105
        path = find_resume_path(args.output_dir, args.resume_from_checkpoint)
        if path is None:
            if rank == 0:
                print(f"Checkpoint '{args.resume_from_checkpoint}' does not exist. Starting a new training run.")
            args.resume_from_checkpoint = None
        else:
            if rank == 0:
                print(f"Resuming from checkpoint {path}")
            global_step = load_state(st, os.path.join(args.output_dir, path), gen)
            assert global_step == int(path.split("-")[1])
    validate = _Validation(args, st, cfg, uncond) if rank == 0 and validation_enabled(args) else None
    gs = gen.get_state()                           # the capture / warm-up batch must not consume the
    st.load_inputs(*next_batch(global_step))       # data stream (resume == uninterrupted run)
    if not args.no_cuda_graph:
        st.capture()
    gen.set_state(gs)
    t0 = time.time()
    first = global_step
    last_loss = None
    while global_step < args.max_train_steps:
        st.load_inputs(*next_batch(global_step))
        lr = _lr_at(args, global_step, world)
        st.set_lr(lr)
        st.step()
        global_step += 1
        if rank == 0 and global_step % args.log_every == 0:
            last_loss = st.loss.item()
            print(json.dumps({"step": global_step, "loss": last_loss, "lr": lr,
                              "steps_per_s": (global_step - first) / (time.time() - t0)}), flush=True)
        if rank == 0 and global_step % args.checkpointing_steps == 0:
            rotate_checkpoints(args.output_dir, args.checkpoints_total_limit)
            save_state(st, cfg, os.path.join(args.output_dir, f"checkpoint-{global_step}"), global_step, gen)
        if validate is not None and global_step % args.validation_steps == 0:
            validate(global_step)
    if world > 1:
        torch.distributed.barrier()               # accelerator.wait_for_everyone()
    if rank == 0:
        save_lora(st, cfg, args.output_dir)
    if world > 1:
        torch.distributed.destroy_process_group()
    return st


def save_lora(st, cfg, out_dir):
    """peft adapter + diffusers `unet_lora/pytorch_lora_weights.safetensors` (T15:924-928, 1378-1382)."""
    from safetensors.torch import save_file
    os.makedirs(os.path.join(out_dir, "unet_lora"), exist_ok=True)
    lora = {k: v.cpu().contiguous() for k, v in st.unet.lora_state_dict().items()}
    save_file(weights.to_peft_keys(lora), os.path.join(out_dir, "adapter_model.safetensors"))
    save_file({"unet." + k: v for k, v in lora.items()}, os.path.join(out_dir, "unet_lora", "pytorch_lora_weights.safetensors"))
    json.dump({"r": cfg.lora_rank, "lora_alpha": cfg.lora_alpha, "target_modules": list(config.LORA_TARGETS),
               "peft_type": "LORA"}, open(os.path.join(out_dir, "adapter_config.json"), "w"))


if __name__ == "__main__":
    main(parse_args())
