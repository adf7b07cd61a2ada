"""Where the benchmark step's GPU time goes: torch.profiler (CUDA activities) over a few replays of the
captured SD1.5 step (bench.py's defaults: bs 8, 512x512, one GPU), in a run of its own (no timing is
taken here; tracing slows the host).  Writes per-kernel totals and per-group totals to OUT_DIR and
prints the card and its power limit, which every number below belongs to.

Usage: python tools/step_profile.py OUT_DIR [--replays N] [--batch 8] [--latent 64]

Groups: gemm (implicit GEMM and its split-K finalize), wgrad, attention forward / backward by kernel
template (d <= 64 wgmma, d > 64 mma.sync), attention delta, group norm, layer norm, elementwise
(GEGLU, upsample, conv_in, casts, adds, PCM math), optimiser (grad norm, AdamW, EMA, LoRA refresh),
other (anything not of this library, e.g. memset / memcpy)."""
import argparse
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

GROUPS = [  # (group, regex on the kernel's name); the first match wins
    ("attn_fwd_wg", r"attn_fwd_wg_kernel"),
    ("attn_bwd_wg", r"attn_bwd_wg_kernel"),
    ("attn_fwd_mma", r"attn_fwd_kernel"),
    ("attn_bwd_mma", r"attn_bwd_(dkdv|dq)_kernel"),
    ("attn_delta", r"attn_delta_kernel"),
    ("gemm", r"pcm_gemm_kernel|splitk_finalize_kernel"),
    ("wgrad", r"pcm_wgrad_kernel"),
    ("groupnorm", r"\bgn_\w+_kernel"),
    ("layernorm", r"\bln_\w+_kernel"),
    ("optimiser", r"sumsq_kernel|adamw_clip_kernel|ema_update_kernel|state_step_kernel|lora_refresh_kernel"),
    ("elementwise", r"geglu_\w+_kernel|upsample2x\w*_kernel|conv3x3_c4_kernel|timestep_embed_kernel|colsum_kernel|"
                    r"add_bf16_kernel|cast_f32_bf16_kernel|pcm_\w+_kernel"),
]


def group_of(name):
    for g, rx in GROUPS:
        if re.search(rx, name):
            return g
    return "other"


def short_name(name):
    """Kernel name without the parameter list; template arguments are kept (they select the variant)."""
    m = re.match(r"(?:void )?([\w:()\s]*?\w+_kernel(?:<[^()]*>)?)", name)
    s = m.group(1) if m else name[:120]
    return re.sub(r"pcm::\(anonymous namespace\)::|pcm::", "", s)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--replays", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--latent", type=int, default=64)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from pcm_b200 import config, weights
    from pcm_b200.step import PCMTrainStep

    if not torch.cuda.is_available():
        raise SystemExit("step_profile: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print(f"card: {gpu}", flush=True)
    cfg = config.SD15
    B, hw = args.batch, args.latent
    sd = weights.synthetic_state_dict(cfg, seed=0)
    step = PCMTrainStep(cfg, sd, dev, batch=B, height=hw, width=hw, multiphase=4, num_ddim_timesteps=50,
                        lr=5e-6, weight_decay=1e-3, max_grad_norm=1.0)
    del sd
    h = bench.synth_batch(cfg, B, hw, seed=100)
    step.load_inputs(h["latents"], h["noise"], h["index"], h["w"], h["prompt"], h["uncond"],
                     text_embeds=h.get("text_embeds"), time_ids=h.get("time_ids"))
    step.capture(warmup=1)
    for _ in range(3):
        step.step()
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.replays):
            step.step()
        torch.cuda.synchronize()

    kernels = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernels.setdefault(short_name(ev.name), {"us": 0.0, "calls": 0})
        k["us"] += ev.device_time
        k["calls"] += 1
    groups = {}
    for name, k in kernels.items():
        g = groups.setdefault(group_of(name), {"us": 0.0, "calls": 0})
        g["us"] += k["us"]
        g["calls"] += k["calls"]
    total = sum(g["us"] for g in groups.values())
    n = args.replays
    os.makedirs(args.out_dir, exist_ok=True)
    rows = sorted(kernels.items(), key=lambda kv: -kv[1]["us"])
    with open(os.path.join(args.out_dir, "kernels.csv"), "w") as f:
        f.write("kernel,group,ms_per_step,calls_per_step,share\n")
        for name, k in rows:
            f.write(f"\"{name}\",{group_of(name)},{k['us'] / n / 1e3:.4f},{k['calls'] / n:g},"
                    f"{k['us'] / total:.4f}\n")
    summary = {"card": gpu, "batch": B, "latent": hw, "replays": n,
               "kernel_ms_per_step": total / n / 1e3,
               "groups": {g: {"ms_per_step": v["us"] / n / 1e3, "calls_per_step": v["calls"] / n,
                              "share": v["us"] / total}
                          for g, v in sorted(groups.items(), key=lambda kv: -kv[1]["us"])}}
    with open(os.path.join(args.out_dir, "groups.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(f"GPU kernel time per step: {total / n / 1e3:.2f} ms (sum of kernel durations over {n} replays)")
    for g, v in summary["groups"].items():
        print(f"  {g:14s} {v['ms_per_step']:8.2f} ms  {100 * v['share']:5.1f} %  {v['calls_per_step']:g} launches")
    print("top kernels (ms per step):")
    for name, k in rows[:15]:
        print(f"  {k['us'] / n / 1e3:8.2f}  {name}")


if __name__ == "__main__":
    main()
