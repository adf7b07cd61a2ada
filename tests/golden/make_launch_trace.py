#!/usr/bin/env python
"""Launch trace of one eager training step (PCMTrainStep.run_eager), recorded on the CPU.

The step runs with ops.DRY_RUN set, so nothing launches.  Every `pcm_gemm` and `pcm_wgrad` descriptor is
recorded field by field, every other C-ABI call with all its arguments, in launch order.  Each record
carries `side`: whether it was enqueued inside UNetB200._Side, the one context manager that moves work to
the weight-gradient stream.  The data-parallel reducer is replaced by a recorder, so the `grad_ready`
bucket signals of the backward appear in sequence too.

Pointers are canonicalised, so two runs compare equal exactly when they issue the same launches on the
same buffers.  Tensor.data_ptr is wrapped for the run: every tensor whose address is taken (by the ops
wrappers, or directly, like the temporaries of PCMTrainStep._teacher_substeps) is kept alive until the
run ends, so the allocator never hands out an address twice, and every address it returns is known to be
one.  A pointer becomes [storage label, byte offset], labels numbered in order of first appearance.

    python tests/golden/make_launch_trace.py                   -> tests/golden/launch_trace.json.gz
    python tests/golden/make_launch_trace.py --config SD15 --batch 1 --hw 8 --out FILE.json.gz
"""
import argparse
import bisect
import ctypes
import gzip
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "launch_trace.json.gz")

# name -> (UNet config, PCMTrainStep keywords); all at batch 2, 16x16 latents
CASES = {
    "TINY": ("TINY", {}),
    "TINY_XL": ("TINY_XL", dict(num_ddim_timesteps=40)),
    "TINY_substeps2_nocfg": ("TINY", dict(teacher_substeps=2, apply_cfg_solver=False)),
    "TINY_ema": ("TINY", dict(ema_decay=0.95)),
}


class Recorder:
    def __init__(self):
        self.keep = []          # registered tensors: alive until the recorder is dropped
        self.starts = []        # sorted storage base addresses
        self.ends = {}          # base -> end address
        self.addrs = set()      # every value Tensor.data_ptr returned
        self.labels = {}        # storage base -> label
        self.trace = []
        self.side = 0

    def register(self, t, p):
        self.keep.append(t)
        self.addrs.add(p)
        s = t.untyped_storage()
        base = s.data_ptr()
        if base not in self.ends:
            bisect.insort(self.starts, base)
            self.ends[base] = base + s.nbytes()

    def ptr(self, p):
        if not p:
            return None
        i = bisect.bisect_right(self.starts, p) - 1
        assert i >= 0 and p <= self.ends[self.starts[i]], f"address {p:#x} of no tensor"
        base = self.starts[i]
        if base not in self.labels:
            self.labels[base] = len(self.labels)
        return [self.labels[base], p - base]

    def emit(self, op, **kw):
        self.trace.append(dict(op=op, side=self.side > 0, **kw))

    def struct(self, s):
        """All fields of a ctypes descriptor; pointers canonicalised, arrays cut to their used length."""
        out = {}
        for name, typ in s._fields_:
            v = getattr(s, name)
            if typ is ctypes.c_void_p:
                out[name] = self.ptr(v)
            elif isinstance(v, ctypes.Structure):
                out[name] = self.struct(v)
            elif isinstance(v, ctypes.Array):
                n = {"a": "num_a", "b": "num_b", "prog": "num_prog"}.get(name, "num_taps")
                out[name] = [self.struct(e) if isinstance(e, ctypes.Structure) else e
                             for e in v[:getattr(s, n)]]
            else:
                out[name] = v
        return out

    def view(self, t):
        return None if t is None else [list(t.shape), list(t.stride()), str(t.dtype).replace("torch.", "")]


def _install(monkeypatch, rec):
    """Route ops' launch wrappers and the side-stream context manager through `rec`."""
    from pcm_b200 import _lib, ops, unet
    descs = []

    class GemmDesc(_lib.GemmDesc):
        def __init__(self):
            super().__init__()
            descs.append(self)

    class WgradDesc(_lib.WgradDesc):
        def __init__(self):
            super().__init__()
            descs.append(self)

    class Side:
        def __init__(self, net, keep):
            pass

        def __enter__(self):
            rec.side += 1
            return self

        def __exit__(self, *a):
            rec.side -= 1
            return False

    gemm, wgrad, call, data_ptr = ops.gemm, ops.wgrad, ops._call, torch.Tensor.data_ptr

    def rec_data_ptr(t):
        p = data_ptr(t)
        rec.register(t, p)
        return p

    def rec_gemm(a_srcs, b_srcs, prog, **kw):
        out = gemm(a_srcs, b_srcs, prog, **kw)
        rec.emit("gemm", desc=rec.struct(descs.pop()), out_view=rec.view(kw["out"]),
                 rowvec_view=rec.view(kw.get("rowvec")), residual_view=rec.view(kw.get("residual")))
        return out

    def rec_wgrad(p_src, q_src, out, **kw):
        res = wgrad(p_src, q_src, out, **kw)
        rec.emit("wgrad", desc=rec.struct(descs.pop()), out_view=rec.view(out))
        return res

    def rec_call(name, *args):
        canon = [rec.ptr(a) if type(a) is int and a in rec.addrs else a for a in args]
        rec.emit(name, args=canon)
        return call(name, *args)

    monkeypatch.setattr(_lib, "GemmDesc", GemmDesc)
    monkeypatch.setattr(_lib, "WgradDesc", WgradDesc)
    monkeypatch.setattr(unet.UNetB200, "_Side", Side)
    monkeypatch.setattr(ops, "gemm", rec_gemm)
    monkeypatch.setattr(ops, "wgrad", rec_wgrad)
    monkeypatch.setattr(ops, "_call", rec_call)
    monkeypatch.setattr(torch.Tensor, "data_ptr", rec_data_ptr)
    monkeypatch.setattr(ops, "_NUM_SMS", 132)
    monkeypatch.setattr(ops, "DRY_RUN", [])


class _Reducer:
    """Stand-in for dp.GradReducer: records start / ready(offset) / finish in sequence."""

    def __init__(self, rec):
        self.rec = rec

    def start(self):
        self.rec.emit("reducer.start")

    def ready(self, off):
        self.rec.emit("reducer.ready", offset=off)

    def finish(self):
        self.rec.emit("reducer.finish")


def record(cfg_name, step_kw, batch=2, hw=16):
    """Canonical launch trace (list of dicts) of one eager step."""
    import pytest
    from pcm_b200 import config, weights
    from pcm_b200.step import PCMTrainStep
    cfg = getattr(config, cfg_name)
    sd = weights.synthetic_state_dict(cfg, 0)
    rec = Recorder()
    with pytest.MonkeyPatch.context() as mp:
        _install(mp, rec)
        st = PCMTrainStep(cfg, sd, "cpu", batch=batch, height=hw, width=hw, multiphase=4, **step_kw)
        st.reducer, st._overlap = _Reducer(rec), True
        rec.trace.clear()
        rec.labels.clear()
        st.run_eager()
    return rec.trace


def dump(traces, path):
    data = json.dumps(traces, sort_keys=True, separators=(",", ":")).encode()
    with open(path, "wb") as f, gzip.GzipFile(fileobj=f, mode="wb", mtime=0, filename="") as z:
        z.write(data)


def load(path):
    with gzip.open(path, "rb") as z:
        return json.loads(z.read())


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", help="one UNet config (e.g. SD15) instead of the committed cases")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--hw", type=int, default=16)
    ap.add_argument("--out", default=FIXTURE)
    a = ap.parse_args()
    cases = {a.config: (a.config, {})} if a.config else CASES
    traces = {}
    for name, (cfg_name, kw) in cases.items():
        traces[name] = record(cfg_name, kw, a.batch, a.hw)
        print(f"{name}: {len(traces[name])} launches")
    dump(traces, a.out)
    print(f"wrote {a.out} ({os.path.getsize(a.out)} bytes)")


if __name__ == "__main__":
    main()
