#!/usr/bin/env python
"""Memory of one PCM-LoRA training step, with and without gradient checkpointing.

    python tools/step_memory.py --model sd15 --batch 8 --latent 64     # GPU: one JSON line
    python tools/step_memory.py --dry-run                              # CPU: the tape table below

On a GPU, for each mode the step is built, captured into a CUDA graph after its eager warm-up (as bench.py
does), run `--warmup` more times and then timed over `--steps` replays with CUDA events.  Reported per mode:
the peak torch.cuda.max_memory_allocated / max_memory_reserved over all of that, steps/s, and the tape
bytes of the eager warm-up step.  A mode that runs out of memory is reported as such (no retry).  The
checkpointed mode runs first, so that an out-of-memory stored-tape run comes last.

--dry-run needs no GPU: the step's host code runs on CPU with ops.DRY_RUN set (kernels are recorded, not
launched) and only the tape is counted, for SD1.5 bs 8 and bs 20 at 64x64 and SDXL bs 2 and bs 4 at
128x128 (or the one configuration given).

Tape bytes are counted over the unique storages reachable from UNetB200.saved just before backward():
  tape_gib          every storage the tape keeps alive;
  row_view_gib      of those, the storages the tape reaches only through a part of them (the student rows
                    of a merged-pass activation keep its whole storage alive);
  block_inputs_gib  the student rows of the block inputs alone (an upsampler's input before the 2x), what
                    the checkpointed tape stores.
"""
import argparse
import dataclasses
import gc
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GIB = float(1 << 30)
DRY_RUN_CASES = [("sd15", 8, 64), ("sd15", 20, 64), ("sdxl", 2, 128), ("sdxl", 4, 128)]


def _tensors(obj, out):
    """Every tensor reachable from a tape (records, lists, dicts, namespaces)."""
    if isinstance(obj, torch.Tensor):
        out.append(obj)
    elif isinstance(obj, dict):
        for v in obj.values():
            _tensors(v, out)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _tensors(v, out)
    elif dataclasses.is_dataclass(obj):
        for f in dataclasses.fields(obj):
            _tensors(getattr(obj, f.name), out)
    elif isinstance(obj, types.SimpleNamespace):
        _tensors(vars(obj), out)
    return out


def _extent(t):
    return t.element_size() * (1 + sum((n - 1) * s for n, s in zip(t.shape, t.stride()))) if t.numel() else 0


def block_inputs(saved):
    """The student rows of every block input on a tape (stored or checkpointed), one entry per tensor."""
    from pcm_b200.unet import CheckpointRec, ResampleRec, ResnetRec, TransformerRec
    seen, out = set(), []
    for blk in saved.tape:
        if isinstance(blk, CheckpointRec):
            xs, div = blk.xs, 1
        elif isinstance(blk, ResnetRec):
            xs, div = blk.norm1.xs, 1
        elif isinstance(blk, TransformerRec):
            xs, div = blk.norm.xs, 1
        elif isinstance(blk, ResampleRec):
            xs, div = blk.conv.xs, 4 if blk.up else 1     # the conv of an upsampler reads the 2x input
        else:
            continue
        for x in xs:
            key = (x.data_ptr(), tuple(x.shape))
            if key not in seen:
                seen.add(key)
                out.append(x.numel() * x.element_size() // div)
    return out


def tape_bytes(saved):
    """{tape_gib, row_view_gib, block_inputs_gib} of UNetB200.saved (see the module docstring)."""
    storages = {}       # storage base -> [nbytes, the largest extent a tape tensor reaches in it]
    for t in _tensors(saved, []):
        s = t.untyped_storage()
        e = storages.setdefault(s.data_ptr(), [s.nbytes(), 0])
        e[1] = max(e[1], t.storage_offset() * t.element_size() + _extent(t))
    total = sum(n for n, _ in storages.values())
    views = sum(n for n, ext in storages.values() if ext < n)
    return dict(tape_gib=round(total / GIB, 3), row_view_gib=round(views / GIB, 3),
                block_inputs_gib=round(sum(block_inputs(saved)) / GIB, 3))


def _measure_tape(step, into):
    """Count the tape of the next backward() of `step` into the dict `into`."""
    net = step.unet
    bwd = net.backward

    def counted(*a, **kw):
        if not into:
            into.update(tape_bytes(net.saved))
        return bwd(*a, **kw)
    net.backward = counted
    return lambda: vars(net).pop("backward", None)


def _config(model):
    from pcm_b200 import config
    return config.SD15 if model == "sd15" else config.SDXL


def _make_step(model, batch, latent, device, ckpt, sd=None):
    from pcm_b200 import weights
    from pcm_b200.step import PCMTrainStep
    cfg = _config(model)
    sd = weights.synthetic_state_dict(cfg, seed=0) if sd is None else sd
    return PCMTrainStep(cfg, sd, device, batch=batch, height=latent, width=latent, multiphase=4,
                        num_ddim_timesteps=50 if model == "sd15" else 40, lr=5e-6, weight_decay=1e-3,
                        max_grad_norm=1.0, gradient_checkpointing=ckpt)


def _inputs(model, batch, latent, seed=100):
    from bench import synth_batch
    h = synth_batch(_config(model), batch, latent, seed=seed, pinned=torch.cuda.is_available())
    return (h["latents"], h["noise"], h["index"], h["w"], h["prompt"], h["uncond"]), \
        dict(text_embeds=h.get("text_embeds"), time_ids=h.get("time_ids"))


def dry_run(model, batch, latent):
    """Tape bytes of both modes, counted on CPU without launching anything."""
    from pcm_b200 import ops, weights
    sd = weights.synthetic_state_dict(_config(model), seed=0)
    out = {}
    old = ops.DRY_RUN
    try:
        for name, ckpt in (("stored_tape", False), ("checkpointed", True)):
            ops.DRY_RUN = []
            st = _make_step(model, batch, latent, "cpu", ckpt, sd)
            a, kw = _inputs(model, batch, latent)
            st.load_inputs(*a, **kw)
            tape = {}
            _measure_tape(st, tape)
            ops.DRY_RUN = []
            st.run_eager()
            out[name] = tape
            del st
            gc.collect()
    finally:
        ops.DRY_RUN = old
    return out


def _gpu_name_and_power():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(pl.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        power = None
    return name, power


def run_gpu(model, batch, latent, ckpt, steps, warmup, sd):
    """One mode on cuda:0: peak memory, steps/s and tape bytes (or the out-of-memory error)."""
    dev = torch.device("cuda", 0)
    torch.zeros(1, device=dev)     # the allocator of a fresh process exists after its first allocation
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    res, st = {}, None
    try:
        st = _make_step(model, batch, latent, dev, ckpt, sd)
        a, kw = _inputs(model, batch, latent)
        st.load_inputs(*a, **kw)
        torch.cuda.synchronize()
        tape = {}
        restore = _measure_tape(st, tape)
        st.capture(warmup=1)
        restore()
        for _ in range(warmup):
            st.step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            st.step()
        e1.record()
        torch.cuda.synchronize()
        res.update(steps_per_s=round(steps * 1e3 / e0.elapsed_time(e1), 4), loss=st.loss.item(), **tape)
    except torch.cuda.OutOfMemoryError as e:
        res.update(oom=True, error=str(e).splitlines()[0][:300])
    res.update(peak_allocated_gib=round((torch.cuda.max_memory_allocated(dev) - base) / GIB, 3),
               peak_reserved_gib=round(torch.cuda.max_memory_reserved(dev) / GIB, 3))
    if st is not None:
        st.graph = st.graph_opt = None
    del st
    gc.collect()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", default=None, choices=["sd15", "sdxl"])
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--latent", type=int, default=None)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dry-run", action="store_true", help="count the tape on CPU, launch nothing")
    args = ap.parse_args()
    if args.dry_run:
        cases = DRY_RUN_CASES if args.model is None else \
            [(args.model, args.batch or 8, args.latent or (64 if args.model == "sd15" else 128))]
        for model, batch, latent in cases:
            print(json.dumps(dict(model=model, batch=batch, latent=latent, dry_run=True,
                                  **dry_run(model, batch, latent))), flush=True)
        return
    model = args.model or "sd15"
    batch = args.batch or 8
    latent = args.latent or (64 if model == "sd15" else 128)
    from pcm_b200 import weights
    sd = weights.synthetic_state_dict(_config(model), seed=0)
    out = {}
    for name, ckpt in (("checkpointed", True), ("stored_tape", False)):
        out[name] = run_gpu(model, batch, latent, ckpt, args.steps, args.warmup, sd)
    gpu, power = _gpu_name_and_power()
    print(json.dumps(dict(model=model, batch=batch, latent=latent, gpu=gpu, power_limit_w=power,
                          steps=args.steps, warmup=args.warmup, **out)), flush=True)


if __name__ == "__main__":
    main()
