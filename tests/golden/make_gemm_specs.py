#!/usr/bin/env python
"""Every distinct `pcm_gemm` / `pcm_wgrad` launch of the real training steps, as pointer-free specs.

One eager step per configuration is dry-run on the CPU (nothing launches) through the Recorder of
make_launch_trace.py; each launch is reduced by tests/gemm_spec.py to a spec, and the first spec of every
launch class (gemm_spec.launch_class) is kept.  tests/test_gemm_prod_gpu.py runs each of them on the GPU
against a float64 reference; tests/test_gemm_specs_cpu.py re-records and compares, so a change to the
launch plan fails on the CPU until the fixture, and with it the GPU suite, holds the new launch.

    python tests/golden/make_gemm_specs.py        -> tests/golden/gemm_specs.json.gz
"""
import dataclasses
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import gemm_spec  # noqa: E402

FIXTURE = os.path.join(HERE, "gemm_specs.json.gz")

# name -> (UNet config, config overrides, PCMTrainStep keywords, batch, latent height = width)
CONFIGS = {
    "SD15_bs8": ("SD15", {}, {}, 8, 64),                       # the benchmark workload
    "SDXL_bs2": ("SDXL", {}, {}, 2, 128),
    "SD15_ckpt": ("SD15", {}, dict(gradient_checkpointing=True), 8, 64),   # the forced merged tiling
    "SD15_rank8": ("SD15", dict(lora_rank=8), {}, 8, 64),      # narrow K chunks, block_n = 32
    "SD15_rank32": ("SD15", dict(lora_rank=32), {}, 8, 64),
}


def record(name):
    """The distinct launch specs of one configuration's eager step."""
    from pcm_b200 import config, weights
    from pcm_b200.step import PCMTrainStep
    cfg_name, over, step_kw, batch, hw = CONFIGS[name]
    cfg = dataclasses.replace(getattr(config, cfg_name), **over)
    sd = weights.synthetic_state_dict(cfg, 0)
    with gemm_spec.recording() as rec:
        st = PCMTrainStep(cfg, sd, "cpu", batch=batch, height=hw, width=hw, multiphase=4, **step_kw)
        rec.trace.clear()
        st.run_eager()
        return gemm_spec.distinct_specs(rec.trace)


def main():
    specs = {}
    for name in CONFIGS:
        specs[name] = record(name)
        print(f"{name}: {len(specs[name])} launch classes "
              f"({sum(s['op'] == 'wgrad' for s in specs[name])} pcm_wgrad, {sum('pre' in s for s in specs[name])} pairs)")
    gemm_spec.trace.dump(specs, FIXTURE)
    print(f"wrote {FIXTURE} ({os.path.getsize(FIXTURE)} bytes)")


if __name__ == "__main__":
    main()
