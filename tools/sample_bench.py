#!/usr/bin/env python
"""Few-step sampler benchmark (pcm_b200/sampling.py): SD1.5 UNet with a rank-64 LoRA (seeded synthetic
weights), 512 x 512 (64 x 64 latents), 4 DDIM-trailing steps.

Reports, on CUDA graph replay: ms per sampler call and images/s at batch 1 and 16 (4 prompts x 4 images),
guidance 1 and 7.5; the time of one LoRA fusion (pcm_lora_fuse over every LoRA target); the fused forward
(lora=False on the fused weights) against the trained network's unfused LoRA forward at the same batch;
peak memory, the GPU name and its power limit.

    python tools/sample_bench.py [--reps 5] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _gpu_info():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    text=True).strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0), "unknown"


def _time(fn, reps):
    """ms per call: CUDA events around `reps` calls after one untimed call."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench needs a CUDA device: there is nothing to measure without one")
    from pcm_b200 import config, weights
    from pcm_b200.sampling import PCMSampler
    from pcm_b200.unet import UNetB200
    dev = torch.device("cuda", 0)
    cfg = config.SD15
    net = UNetB200(cfg, weights.synthetic_state_dict(cfg, 0), dev, need_backward=False)
    torch.cuda.synchronize()
    s = PCMSampler(net)
    out = {"model": "sd15", "resolution": 512, "steps": args.steps, "lora_rank": cfg.lora_rank}
    out["fuse_ms"] = _time(lambda: s.fuse(), args.reps)
    fused_bytes = 2 * 2 * s.net.fused_weights.numel()
    out["fuse_GBps"] = fused_bytes / (out["fuse_ms"] * 1e-3) / 1e9
    g = torch.Generator().manual_seed(0)
    runs = []
    for P, nipp in ((1, 1), (4, 4)):
        pe = torch.randn(P, 77, 768, generator=g)
        ne = torch.randn(P, 77, 768, generator=g)
        for gs in (1.0, 7.5):
            gen = torch.Generator(device=dev).manual_seed(0)

            def call():
                return s(pe, ne, num_inference_steps=args.steps, guidance_scale=gs, num_images_per_prompt=nipp,
                         height=512, width=512, generator=gen)
            ms = _time(call, args.reps)
            B = P * nipp
            runs.append(dict(batch=B, guidance=gs, unet_batch=2 * B if gs > 1 else B, ms_per_call=ms,
                             images_per_s=B / (ms * 1e-3)))
            print(json.dumps(runs[-1]), flush=True)
    out["sampling"] = runs
    # fused vs unfused LoRA forward at the same batch (eager, one forward each)
    fwd = []
    for B in (2, 16):
        x = torch.randn(B, 64, 64, 4, generator=g).to(dev)
        t = torch.full((B,), 999, device=dev)
        ctx = torch.randn(B * 77, 768, generator=g).to(dev, torch.bfloat16)
        unf = _time(lambda: net.forward(x, t, ctx, lora=True), args.reps)
        fus = _time(lambda: s.net.forward(x, t, ctx, lora=False), args.reps)
        fwd.append(dict(batch=B, unfused_lora_ms=unf, fused_ms=fus, speedup=unf / fus))
    out["forward"] = fwd
    out["peak_mem_GiB"] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    out["gpu"], out["power_limit"] = _gpu_info()
    line = json.dumps(out)
    print(line, flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
