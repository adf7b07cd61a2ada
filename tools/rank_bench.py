"""Training-step speed and memory per LoRA rank on the SD1.5 benchmark shape (bs 8, 512x512 -> 64x64
latents, CUDA-graph captured, one GPU): steps/s, peak memory of the step (above what was allocated before it), and the GPU time of the implicit GEMM and
of the LoRA weight gradients per step, for each `--ranks` value.

Two steps fit on an 80 GB card, not five: the r = 64 step stays resident and each other rank is built in
turn and timed in `--rounds` runs alternated with r = 64, so a drift of the card's clock affects both
alike (the table gives each rank's speed relative to its own interleaved r = 64 runs); the card's name and
power limit are read at the start of the same run and printed with the table.  Kernel totals come from a separate torch.profiler
pass over a few replays (tracing slows the host, so it is not part of the timed runs).

Usage: python tools/rank_bench.py [--ranks 8 16 32 64 128] [--steps 20] [--warmup 5] [--rounds 3]"""
import argparse
import dataclasses
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[8, 16, 32, 64, 128])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--replays", type=int, default=3, help="profiled replays per rank (kernel totals)")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--latent", type=int, default=64)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from pcm_b200 import config, weights
    from pcm_b200.step import PCMTrainStep
    from step_profile import card, group_of, short_name

    if not torch.cuda.is_available():
        raise SystemExit("rank_bench: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print(f"card: {gpu}", flush=True)
    B, hw = args.batch, args.latent
    h = bench.synth_batch(config.SD15, B, hw, seed=100)
    peak, times, kern = {}, {}, {}

    def build(r):
        cfg = dataclasses.replace(config.SD15, lora_rank=r)
        sd = weights.synthetic_state_dict(cfg, seed=0)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        st = PCMTrainStep(cfg, sd, dev, batch=B, height=hw, width=hw, multiphase=4, num_ddim_timesteps=50,
                          lr=5e-6, weight_decay=1e-3, max_grad_norm=1.0)
        del sd
        st.load_inputs(h["latents"], h["noise"], h["index"], h["w"], h["prompt"], h["uncond"])
        st.capture(warmup=1)
        for _ in range(args.warmup):
            st.step()
        torch.cuda.synchronize()
        peak[r] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 30
        return st

    def timed(st):
        st.step()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            st.step()
        torch.cuda.synchronize()
        return args.steps / (time.perf_counter() - t0)

    def kernels(st):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.replays):
                st.step()
            torch.cuda.synchronize()
        tot = {"gemm": 0.0, "wgrad": 0.0}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                g = group_of(short_name(ev.name))
                if g in tot:
                    tot[g] += ev.device_time / args.replays / 1e3
        return tot

    ref = build(64)
    kern[64] = kernels(ref)
    times[64] = []
    rel = {}
    for r in args.ranks:
        if r == 64:
            continue
        st = build(r)
        times[r], t64 = [], []
        for _ in range(args.rounds):     # alternate with the resident r = 64 step
            times[r].append(timed(st))
            t64.append(timed(ref))
        times[64] += t64
        rel[r] = sorted(a / b for a, b in zip(times[r], t64))[len(t64) // 2]
        kern[r] = kernels(st)
        del st
        torch.cuda.empty_cache()
    rel[64] = 1.0
    rows = []
    print(f"SD1.5 bs {B}, {hw * 8}x{hw * 8}, graph-captured, {args.rounds} alternated rounds of {args.steps} steps")
    print("| r | steps/s (median; min-max) | vs interleaved r = 64 | peak GiB | GEMM ms/step | wgrad ms/step |")
    print("|---|---|---|---|---|---|")
    for r in args.ranks:
        t = sorted(times[r])
        row = dict(r=r, steps_per_s=t[len(t) // 2], spread=[t[0], t[-1]], vs_r64=rel[r], peak_gib=peak[r],
                   gemm_ms=kern[r]["gemm"], wgrad_ms=kern[r]["wgrad"])
        rows.append(row)
        print(f"| {r} | {row['steps_per_s']:.3f} ({t[0]:.3f}-{t[-1]:.3f}) | {rel[r]:.3f} | {peak[r]:.2f} | "
              f"{row['gemm_ms']:.1f} | {row['wgrad_ms']:.1f} |")
    print(json.dumps({"card": gpu, "rows": rows}))


if __name__ == "__main__":
    main()
