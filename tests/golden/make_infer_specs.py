#!/usr/bin/env python
"""Every distinct GEMM and glue launch of the two inference paths - the VAE and the few-step sampler - as
pointer-free specs.

Each configuration is built (seeded synthetic weights) and then dry-run on the CPU (nothing launches)
through tests/op_spec.py's recording(); the first spec of every GEMM launch class (gemm_spec.launch_class)
and of every covered op's launch class (op_spec.launch_class) is kept.  Recording starts after
construction, so the sampler's LoRA fuse (tests/test_sampler_gpu.py) is not part of it.  On the GPU the
sampler captures the same launches into a CUDA graph; here it runs them eagerly.
tests/test_infer_prod_gpu.py runs each new class on the GPU against a float64 reference;
tests/test_infer_specs_cpu.py re-records and compares, so a change to either inference plan fails on the
CPU until the fixture, and with it the GPU suite, holds the new launch.

    python tests/golden/make_infer_specs.py        -> tests/golden/infer_specs.json.gz
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import gemm_spec  # noqa: E402
import op_spec  # noqa: E402

FIXTURE = os.path.join(HERE, "infer_specs.json.gz")
SDXL_SCALING = 0.13025

# VAE: name -> (VAE config overrides, "encode" / "decode", batch, image height, image width, outputs of
# the image exit: "f32" NCHW fp32, "u8" uint8 NHWC)
VAE_CONFIGS = {
    "vae_sd15_enc512_b8": ({}, "encode", 8, 512, 512, None),
    # the trainer's --validation_images decode: 4 prompts x 4 images, exactly MAX_LAUNCH_ELEMENTS
    "vae_sd15_dec512_b16": ({}, "decode", 16, 512, 512, ("u8",)),
    "vae_sd15_dec512_b17": ({}, "decode", 17, 512, 512, ("f32", "u8")),      # a sub-batch of 16, then 1
    "vae_sdxl_enc1024_b1": (dict(scaling_factor=SDXL_SCALING), "encode", 1, 1024, 1024, None),
    "vae_sdxl_dec1024_b4": (dict(scaling_factor=SDXL_SCALING), "decode", 4, 1024, 1024, ("f32", "u8")),
    # mid-block S = 33 x 32 = 1056 tokens: a narrow last K chunk for P V, M no multiple of 128
    "vae_sd15_enc264x256_b1": ({}, "encode", 1, 264, 256, None),
    "vae_sd15_dec264x256_b1": ({}, "decode", 1, 264, 256, ("f32",)),
    # S = 96 x 128 = 12288 tokens: query chunks of 2688 rows, the last one ragged (1536 rows)
    "vae_sd15_dec768x1024_b1": ({}, "decode", 1, 768, 1024, ("u8",)),
}
# sampler: name -> (UNet config, image side, guidance scale, output_type); one prompt, 4 images per prompt,
# as the trainer's validation samples
SAMPLER_CONFIGS = {
    "sampler_sd15_512_g1": ("SD15", 512, 1.0, "latent"),             # UNet batch 4
    "sampler_sd15_512_g7.5": ("SD15", 512, 7.5, "latent"),           # UNet batch 8 ([uncond; cond])
    "sampler_sdxl_1024_g1": ("SDXL", 1024, 1.0, "latent"),
    "sampler_sd15_512_g1_pt": ("SD15", 512, 1.0, "pt"),              # the VAE decode inside the sampling loop
}
CONFIGS = list(VAE_CONFIGS) + list(SAMPLER_CONFIGS)
NUM_INFERENCE_STEPS = 2
IMAGES_PER_PROMPT = 4


def _vae(over):
    from pcm_b200 import vae
    return vae.AutoencoderKL.from_pretrained(None, device="cpu", config=dict(over), seed=0)


def _record_vae(name):
    over, what, B, H, W, outs = VAE_CONFIGS[name]
    with op_spec.recording() as rec:
        v = _vae(over)
        rec.trace.clear()
        if what == "encode":
            v.encode(torch.zeros(B, 3, H, W)).latent_dist.sample(torch.Generator().manual_seed(0))
        else:
            n = len(v.cfg.block_out_channels) - 1
            z = torch.zeros(B, H >> n, W >> n, 4)
            out = torch.empty(B, 3, H, W) if "f32" in outs else None
            u8 = torch.empty(B, H, W, 3, dtype=torch.uint8) if "u8" in outs else None
            v.decode_images(z, v.cfg.scaling_factor, out, u8)
        return rec.trace


def _record_sampler(name):
    from pcm_b200 import config, weights
    from pcm_b200.sampling import PCMSampler
    from pcm_b200.unet import UNetB200
    cfg_name, side, g, output_type = SAMPLER_CONFIGS[name]
    cfg = getattr(config, cfg_name)
    with op_spec.recording() as rec:
        net = UNetB200(cfg, weights.synthetic_state_dict(cfg, 0), "cpu", need_backward=False)
        smp = PCMSampler(net, vae=_vae({}) if output_type != "latent" else None)
        rec.trace.clear()
        pe = torch.zeros(1, 77, cfg.cross_attention_dim)
        kw = {}
        if cfg.addition_embed:
            te = torch.zeros(1, cfg.text_embed_dim)
            kw = dict(text_embeds=te, time_ids=torch.tensor([side, side, 0, 0, side, side]), negative_text_embeds=te)
        smp(pe, torch.zeros_like(pe), num_inference_steps=NUM_INFERENCE_STEPS, guidance_scale=g,
            num_images_per_prompt=IMAGES_PER_PROMPT, height=side, width=side, generator=torch.Generator().manual_seed(0),
            output_type=output_type, **kw)
        return rec.trace


def record_trace(name):
    """The whole launch trace (every `_call` record and every GEMM descriptor) of one configuration."""
    return _record_vae(name) if name in VAE_CONFIGS else _record_sampler(name)


def distinct(records):
    """{"gemm": first spec of every GEMM launch class, "ops": of every covered op's launch class}."""
    return dict(gemm=gemm_spec.distinct_specs(records), ops=op_spec.distinct_specs(records))


def main():
    specs = {}
    for name in CONFIGS:
        specs[name] = distinct(record_trace(name))
        big = max(s["desc"]["M"] * s["desc"]["N"] for s in specs[name]["gemm"])
        print(f"{name}: {len(specs[name]['gemm'])} GEMM classes (largest M N = {big}), "
              f"{len(specs[name]['ops'])} op classes")
    op_spec.trace.dump(specs, FIXTURE)
    print(f"wrote {FIXTURE} ({os.path.getsize(FIXTURE)} bytes)")


if __name__ == "__main__":
    main()
