#!/usr/bin/env python
"""Golden vectors of the reference's flow-matching solver / schedulers, produced by EXECUTING the
reference classes verbatim (AST-extracted from the read-only tree; the diffusers mixins they inherit
from are replaced by empty stand-ins, which only provide `.config`):

    EulerSolver                   $PCM_REFERENCE/code/text_to_image_sd3/train_pcm_lora_sd3.py:160-226
    PCMFMDeterministicScheduler   .../pcm_fm_deterministic_scheduler.py:35-242
    PCMFMStochasticScheduler      .../pcm_fm_stochastic_scheduler.py:35-243

    python tests/golden/make_fm_golden.py   ->  tests/golden/fm_math.pt
"""
import ast
import os
import types

import numpy as np
import torch

# a checkout of G-U-N/Phased-Consistency-Model (read only), given by PCM_REFERENCE
REF = os.path.join(os.environ["PCM_REFERENCE"], "code/text_to_image_sd3")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fm_math.pt")


def extract(path, names):
    src = open(path).read()
    lines = src.splitlines()
    tree = ast.parse(src)
    parts = []
    for n in tree.body:
        if isinstance(n, (ast.ClassDef, ast.FunctionDef)) and n.name in names:
            first = min([n.lineno] + [d.lineno for d in n.decorator_list])   # keep decorators (@dataclass)
            parts.append("\n".join(lines[first - 1:n.end_lineno]))
    return "\n\n".join(parts)


class ConfigMixin:
    pass


class SchedulerMixin:
    pass


class BaseOutput:
    pass


def register_to_config(init):
    def wrapped(self, **kw):
        import inspect
        sig = inspect.signature(init)
        cfg = {k: v.default for k, v in sig.parameters.items() if k != "self"}
        cfg.update(kw)
        self.config = types.SimpleNamespace(**cfg)
        init(self, **cfg)
    return wrapped


def namespace():
    from dataclasses import dataclass
    from typing import Optional, Tuple, Union
    return dict(np=np, torch=torch, dataclass=dataclass, Optional=Optional, Tuple=Tuple, Union=Union,
                ConfigMixin=ConfigMixin, SchedulerMixin=SchedulerMixin, BaseOutput=BaseOutput,
                register_to_config=register_to_config, print=lambda *a, **k: None)


def main():
    ns = namespace()
    exec(extract(os.path.join(REF, "train_pcm_lora_sd3.py"), {"extract_into_tensor", "EulerSolver"}), ns)
    exec(extract(os.path.join(REF, "pcm_fm_deterministic_scheduler.py"),
                 {"PCMFMDeterministicSchedulerOutput", "PCMFMDeterministicScheduler"}), ns)
    exec(extract(os.path.join(REF, "pcm_fm_stochastic_scheduler.py"),
                 {"PCMFMStochasticSchedulerOutput", "PCMFMStochasticScheduler"}), ns)
    g = torch.Generator().manual_seed(0)
    out = {}
    # ---- EulerSolver (training) : sigmas of the SD3 scheduler, shift 3.0 (T3:1040-1050) -----------
    shift = 3.0
    t = np.linspace(1, 1000, 1000, dtype=np.float32)[::-1].copy()
    sig = t / 1000
    sig = (shift * sig / (1 + (shift - 1) * sig)).astype(np.float32)
    sigmas_train = sig[::-1].copy()                      # ascending, as the script feeds the solver
    out["sigmas_train"] = torch.from_numpy(sigmas_train)
    solver = ns["EulerSolver"](sigmas_train, 1000, 50)
    out["euler"] = dict(euler_timesteps=solver.euler_timesteps, euler_timesteps_prev=solver.euler_timesteps_prev,
                        sigmas=solver.sigmas, sigmas_prev=solver.sigmas_prev)
    B = 8
    x = torch.randn(B, 4, 4, 4, generator=g)
    v = torch.randn(B, 4, 4, 4, generator=g)
    idx = torch.tensor([0, 5, 12, 13, 24, 25, 37, 49])
    out["x"], out["v"], out["idx"] = x, v, idx
    out["euler_step"] = solver.euler_step(x, v, idx)
    for mp in (1, 2, 4):
        for tgt in (False, True):
            xp, end = solver.euler_style_multiphase_pred(x, v, idx, mp, is_target=tgt)
            out[f"euler_mp{mp}_{int(tgt)}"] = (xp, end)
    # ---- inference schedulers ---------------------------------------------------------------
    noise = torch.randn(B, 4, 4, 4, generator=g)
    out["noise"] = noise
    for name, cls in (("det", ns["PCMFMDeterministicScheduler"]), ("sto", ns["PCMFMStochasticScheduler"])):
        for shift in (1.0, 3.0):
            for n in (1, 2, 4, 8):
                s = cls(num_train_timesteps=1000, shift=shift, pcm_timesteps=50)
                rec = dict(sigmas=s.sigmas.clone(), timesteps0=s.timesteps.clone(), sigma_min=s.sigma_min,
                           sigma_max=s.sigma_max)
                s.set_timesteps(n)
                rec["timesteps"] = s.timesteps.clone()
                rec["sigmas_"] = s.sigmas_.clone()
                cur = x.clone()
                steps = []
                for i, ts in enumerate(s.timesteps):
                    torch.manual_seed(100 + i)           # the stochastic step draws torch.randn_like
                    z = torch.randn_like(cur)
                    torch.manual_seed(100 + i)
                    cur = s.step(v * (1 + 0.1 * i), ts, cur).prev_sample
                    steps.append((cur.clone(), z))
                rec["steps"] = steps
                s2 = cls(num_train_timesteps=1000, shift=shift, pcm_timesteps=50)
                s2.set_timesteps(n)
                rec["scale_noise"] = s2.scale_noise(x, s2.timesteps[0], noise)
                out[f"{name}_shift{shift}_n{n}"] = rec
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
