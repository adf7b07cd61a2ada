"""Time the CUDA VAE (pcm_b200/vae.py): encode and decode of 1 and 16 images at 512^2 and 4 images at 1024^2,
graph-replayed after warm-up, timed with CUDA events.  Prints one JSON line per case with the time per call,
TFLOP/s from the shape-derived FLOP count below, the peak max_memory_allocated, and the card's name and power
limit read in the same run.

    python tools/vae_bench.py [--iters 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def flops(cfg, H, W):
    """(encode, decode) FLOPs of one image: 2 x MACs of every convolution, Linear and attention product."""
    ch, lpb = cfg.block_out_channels, cfg.layers_per_block
    total = {"e": 0.0, "d": 0.0}

    def conv(k, cin, cout, h, w, part):
        total[part] += 2.0 * k * k * cin * cout * h * w

    def res(cin, cout, h, w, part):
        conv(3, cin, cout, h, w, part)
        conv(3, cout, cout, h, w, part)
        if cin != cout:
            conv(1, cin, cout, h, w, part)

    def mid(c, h, w, part):
        res(c, c, h, w, part)
        S = h * w
        total[part] += 4 * 2.0 * S * c * c + 2 * 2.0 * S * S * c
        res(c, c, h, w, part)

    h, w = H, W
    conv(3, 3, ch[0], h, w, "e")
    cin = ch[0]
    for i, c in enumerate(ch):
        for _ in range(lpb):
            res(cin, c, h, w, "e")
            cin = c
        if i < len(ch) - 1:
            h, w = h // 2, w // 2
            conv(3, c, c, h, w, "e")
    mid(ch[-1], h, w, "e")
    conv(3, ch[-1], 8, h, w, "e")
    conv(1, 8, 8, h, w, "e")
    conv(1, 4, 4, h, w, "d")
    conv(3, 4, ch[-1], h, w, "d")
    mid(ch[-1], h, w, "d")
    cin = ch[-1]
    for i, c in enumerate(reversed(ch)):
        for _ in range(lpb + 1):
            res(cin, c, h, w, "d")
            cin = c
        if i < len(ch) - 1:
            h, w = 2 * h, 2 * w
            conv(3, c, c, h, w, "d")
    conv(3, ch[0], 3, h, w, "d")
    return total["e"], total["d"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from pcm_b200 import vae
    if not torch.cuda.is_available():
        raise SystemExit("vae_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(dev)
    v = vae.AutoencoderKL.from_pretrained(None, device=dev, seed=0)
    results = []
    for B, S in ((1, 512), (16, 512), (4, 1024)):
        fe, fd = flops(v.cfg, S, S)
        images = torch.rand(B, 3, S, S, device=dev) * 2 - 1
        x4 = torch.zeros(B, S, S, 4, device=dev)
        x4[..., :3] = images.permute(0, 2, 3, 1)
        z = torch.randn(B, S // 8, S // 8, 4, device=dev)
        img = torch.empty(B, 3, S, S, device=dev)
        cases = [("encode", lambda: v.encode_nhwc(x4), fe),
                 ("decode", lambda: v.decode_images(z, v.config.scaling_factor, img), fd)]
        for name, fn, fl in cases:
            if name == "encode" and B * S * S * max(v.cfg.block_out_channels[:2]) > vae.MAX_LAUNCH_ELEMENTS:
                continue
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn()
                fn()
            torch.cuda.current_stream().wait_stream(s)
            v._hold_workspaces()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                fn()
            g.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.iters
            r = dict(case=f"{name} {B} x {S}^2", ms=round(ms, 3), tflop=round(B * fl / 1e12, 3),
                     tflops=round(B * fl / ms / 1e9, 1), peak_gib=round(torch.cuda.max_memory_allocated() / 2**30, 2),
                     card=card)
            print(json.dumps(r), flush=True)
            results.append(r)
            del g
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
