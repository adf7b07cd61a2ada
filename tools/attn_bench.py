"""Micro-benchmark of pcm_attn_fwd / pcm_attn_bwd on the step's attention shapes (CUDA events).

The forward and the whole backward are timed with CUDA events around back-to-back calls; the backward's
split into its kernels (delta, dK / dV, dQ) comes from a torch.profiler run of its own over the same calls.
--dump DIR writes, at every shape, the outputs (out, lse, dq, dk, dv) of seeded inputs as .npy (bf16 as
its raw int16 bits), so that two builds can be compared bit for bit with --compare DIR_A DIR_B.

Usage: python tools/attn_bench.py [--dump DIR] [--iters N]
       python tools/attn_bench.py --compare DIR_A DIR_B"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [  # (B, H, Sq, Skv, D); the backward runs at B = 8 (the step's backward batch)
    # SD1.5 (bs 8: the merged forward runs 24 samples): 64x64, 32x32, 16x16 latents, cross-attention
    (24, 8, 4096, 4096, 40), (8, 8, 4096, 4096, 40), (24, 8, 4096, 77, 40), (8, 8, 4096, 77, 40),
    (24, 8, 1024, 1024, 80), (8, 8, 1024, 1024, 80), (24, 8, 256, 256, 160),
    # SDXL d = 64: 10 heads at 64x64, 20 heads at 32x32, cross-attention
    (8, 10, 4096, 4096, 64), (8, 20, 1024, 1024, 64), (8, 10, 4096, 77, 64),
]

def shape_id(s):
    return "B{}_H{}_Sq{}_Skv{}_D{}".format(*s)


def compare(a, b):
    import numpy as np
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    assert names, f"no .npy files in {a}"
    bad = 0
    for n in names:
        x, y = np.load(os.path.join(a, n)), np.load(os.path.join(b, n))
        same = x.shape == y.shape and x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8))
        if not same:
            bad += 1
            diff = int((x != y).sum()) if x.shape == y.shape else -1
            print(f"DIFFERENT {n}: {diff} of {x.size} elements")
    missing = sorted(set(f for f in os.listdir(b) if f.endswith(".npy")) - set(names))
    for n in missing:
        print(f"MISSING in {a}: {n}")
    print(f"{len(names) - bad} of {len(names)} files bitwise identical" + (f", {len(missing)} missing" if missing else ""))
    return bad == 0 and not missing


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=int(os.environ.get("ITERS", "10")))
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"), default=None)
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from pcm_b200 import ops

    dev = torch.device("cuda")
    BF = torch.bfloat16
    iters = args.iters
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)

    def timeit(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / iters

    def kernel_split(fn):
        """Mean device time per call of each kernel fn launches (a profiled run of its own)."""
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fn()
            torch.cuda.synchronize()
        t = {}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            n = ev.name
            key = ("dkdv" if "attn_bwd_wg_kernel<true" in n or "attn_bwd_dkdv_kernel" in n else
                   "dq" if "attn_bwd_wg_kernel<false" in n or "attn_bwd_dq_kernel" in n else
                   "delta" if "attn_delta_kernel" in n else "other")
            t[key] = t.get(key, 0.0) + ev.device_time / iters
        return t

    for si, (B, H, Sq, Skv, D) in enumerate(SHAPES):
        C = H * D
        g = torch.Generator(device=dev).manual_seed(1000 + si)
        rnd = lambda r: torch.randn(r, C, device=dev, generator=g).to(BF)
        q, k, v, do = rnd(B * Sq), rnd(B * Skv), rnd(B * Skv), rnd(B * Sq)
        o = torch.empty_like(q)
        lse = torch.empty(B, H, Sq, device=dev, dtype=torch.float32)
        delta = torch.empty_like(lse)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        sc = D ** -0.5
        fwd = lambda: ops.attn_fwd(q, k, v, o, lse, B, H, Sq, Skv, D, sc)
        bwd = lambda: ops.attn_bwd(q, k, v, o, do, lse, delta, dq, dk, dv, B, H, Sq, Skv, D, sc)
        tf = timeit(fwd)
        fl = 4.0 * B * H * Sq * Skv * D
        line = f"B={B} H={H} Sq={Sq} Skv={Skv} D={D}: fwd {tf:8.1f} us {fl / tf / 1e6:7.1f} TFLOP/s"
        if B == 8:
            tb = timeit(bwd)
            sp = kernel_split(bwd)
            line += (f" | bwd {tb:8.1f} us {2.5 * fl / tb / 1e6:7.1f} TFLOP/s"
                     f" (dkdv {sp.get('dkdv', 0):7.1f} us, dq {sp.get('dq', 0):7.1f} us,"
                     f" delta {sp.get('delta', 0):5.1f} us)")
        print(line, flush=True)
        if args.dump:
            fwd()
            outs = dict(out=o, lse=lse)
            if B == 8:
                bwd()
                outs.update(dq=dq, dk=dk, dv=dv)
            torch.cuda.synchronize()
            for n, t in outs.items():
                a = t.view(torch.int16) if t.dtype == BF else t
                np.save(os.path.join(args.dump, f"{shape_id((B, H, Sq, Skv, D))}_{n}.npy"), a.cpu().numpy())
        del q, k, v, do, o, lse, delta, dq, dk, dv
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
