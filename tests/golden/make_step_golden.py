#!/usr/bin/env python
"""Golden vectors of the oracle step (oracle/pcm_ref.py::pcm_step_ref over oracle/unet_ref.py) at the
BASELINE configurations, generated on the CPU in this container (no GPU needed):

    config 1  SD1.5 UNet, bs 1, 32x32 latents, 2-phase      (the reference's CPU smoke case)
    config 2  SD1.5 UNet, bs 8, 64x64 latents, 4-phase      (the benchmark workload of bench.py)

each in two oracle modes: `fp32` (the reference's real CPU semantics: torch.autocast is a no-op
without CUDA, T15:1139-1293 run in fp32) and `bf16` (emulate_bf16=True: weights and every tensor the
reference materialises under bf16 autocast rounded to bf16).  Seeded synthetic weights
(unet_ref.init_params(SD15, 0), LoRA B ~ N(0, 0.02)) and inputs (pcm_ref.make_batch(seed=0)); a
checksum of the weights is stored so the GPU test can verify it regenerated the same parameters.
Tensors larger than SAMPLE elements (config 2) are stored as a fixed, seeded sample of flat NCHW
positions (`sample_idx`, the same positions for every tensor) so that each file stays well under 1 MB.

    python tests/golden/make_step_golden.py [1] [2]      ->  tests/golden/step_config{1,2}.pt
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import pcm_ref, unet_ref  # noqa: E402

CONFIGS = {1: dict(B=1, hw=32, multiphase=2), 2: dict(B=8, hw=64, multiphase=4)}
SAMPLE = 16384
TENSORS = ("eps_student", "x_prev", "model_pred", "target", "noisy")


def sample_tensors(out):
    """Replace every stored latent-shaped tensor by its values at `sample_idx` when it has more than
    SAMPLE elements (seeded positions, sorted)."""
    n = out["bf16"]["x_prev"].numel()
    if n <= SAMPLE:
        return out
    g = torch.Generator().manual_seed(20240)
    idx = torch.randperm(n, generator=g)[:SAMPLE].sort().values
    out["sample_idx"] = idx.to(torch.int32)
    for mode in ("fp32", "bf16"):
        for k in TENSORS:
            if k in out[mode]:
                out[mode][k] = out[mode][k].reshape(-1)[idx].clone()
    return out


def param_checksum(P):
    """Order-independent fingerprint of the seeded weights (double sums of a few statistics)."""
    s1 = sum(v.double().sum().item() for v in P.values())
    s2 = sum((v.double() ** 2).sum().item() for v in P.values())
    return torch.tensor([s1, s2, float(sum(v.numel() for v in P.values()))], dtype=torch.float64)


def main():
    which = [int(a) for a in sys.argv[1:]] or [1, 2]
    cfg = unet_ref.SD15
    P = unet_ref.init_params(cfg, 0)
    for c in which:
        kw = CONFIGS[c]
        batch = pcm_ref.make_batch(cfg, kw["B"], kw["hw"], seed=0)
        out = dict(config=kw, param_checksum=param_checksum(P), index=batch["index"], w=batch["w"])
        for mode, emu in (("fp32", False), ("bf16", True)):
            t0 = time.time()
            with torch.no_grad():
                r = pcm_ref.pcm_step_ref(cfg, P, batch, multiphase=kw["multiphase"], emulate_bf16=emu,
                                         need_grad=False)
            print(f"config {c} {mode}: loss {r['loss'].item():.8f}  ({time.time() - t0:.0f} s)", flush=True)
            out[mode] = dict(loss=r["loss"].double(), eps_student=r["eps_student"].float(),
                             x_prev=r["x_prev"].float(), model_pred=r["model_pred"].float(),
                             target=r["target"].float(),
                             start_timesteps=r["start_timesteps"], timesteps=r["timesteps"],
                             end_timesteps=r["end_timesteps"])
            if emu:
                out[mode]["noisy"] = r["noisy"].float()     # bit-exact target of pcm_add_noise
        torch.save(sample_tensors(out), os.path.join(ROOT, "tests", "golden", f"step_config{c}.pt"))


if __name__ == "__main__":
    main()
