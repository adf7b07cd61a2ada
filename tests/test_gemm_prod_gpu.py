"""Every distinct pcm_gemm / pcm_wgrad launch of the real training steps, on the GPU against float64.

tests/golden/gemm_specs.json.gz holds one pointer-free spec per launch class of the SD1.5 (batch 8, 64x64
latents: the benchmark), SDXL, gradient-checkpointing and rank 8 / 32 steps; test_gemm_specs_cpu.py keeps it
equal to the plan.  Each class is materialised into NaN-poisoned buffers, launched through the C ABI exactly
as recorded (same block_n, ksplit, strides, dep_a_src1; a dep_a_src1 launch back to back after the LoRA
down-projection that writes its poisoned intermediate), compared elementwise with gemm_spec.reference
under gemm_spec.bound, and every byte outside the destination window must be unchanged.  A class met in
several configurations runs once."""
import ctypes
import os
import time

import pytest
import torch

import gemm_cases
import gemm_spec as G
from gemm_cases import restore, result, run_and_check

pytestmark = pytest.mark.gpu

_SPECS = G.trace.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_specs.json.gz"))
CLASSES, COUNTS = {}, {}
for _name, _specs in _SPECS.items():
    COUNTS[_name] = len(_specs)
    for _i, _s in enumerate(_specs):
        CLASSES.setdefault(G.launch_class(_s), (f"{_name}-{_i}", _s))
CASES = list(CLASSES.values())
T0 = time.time()


@pytest.mark.parametrize("spec", [c[1] for c in CASES], ids=[c[0] for c in CASES])
def test_production_launch(cuda, spec):
    T = G.materialise(spec, cuda, seed=len(spec["spans"]))
    before = G.snapshot(T)
    d = spec["desc"]
    if spec["op"] == "wgrad":
        run_and_check(spec, T, before)                       # unordered atomics: within the bound
        restore(T, before)
        o1 = run_and_check(spec, T, before, sem=True)        # turnstile: bit-reproducible
        restore(T, before)
        o2 = run_and_check(spec, T, before, sem=True)
        assert torch.equal(o1, o2)
        assert not T.sem.any(), "the kernel must leave the semaphores at zero"
        return
    if "pre" in spec:                                        # the pair, with the intermediate poisoned
        flat, idx = G.window(dict(op="gemm", desc=spec["pre"]), T)
        assert flat[idx].isnan().all()
    o1 = run_and_check(spec, T, before)
    if G.resolved_ksplit(d) > 1:             # bit-reproducible: the slices are added in split order
        restore(T, before)
        T.ws.fill_(float("nan"))
        G.launch(spec, T)
        assert torch.equal(o1.view(torch.int16 if not d["out_fp32"] else torch.int32),
                           result(spec, T).view(torch.int16 if not d["out_fp32"] else torch.int32))
    kb = [i for i, b in enumerate(d["b"]) if b["kblocked"]]
    if kb:      # K-blocked storage is a pure re-layout: row-major copies of the same weights, bit-identical output
        restore(T, before)
        rows = {i: T.bsrc(d["b"][i]).contiguous() for i in kb}
        from pcm_b200 import _lib
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if "pre" in spec:
            dp = G.gemm_desc(spec["pre"], T, ws=T.ws_pre)
            _lib.check(_lib.lib().pcm_gemm(ctypes.byref(dp), st), "pcm_gemm")
        s = G.gemm_desc(d, T)
        for i, w in rows.items():
            s.b[i].ptr, s.b[i].ld, s.b[i].kblocked = w.data_ptr(), w.shape[1], 0
        _lib.check(_lib.lib().pcm_gemm(ctypes.byref(s), st), "pcm_gemm")
        torch.cuda.synchronize()
        o2 = result(spec, T)
        assert torch.equal(o1.view(torch.int16 if not d["out_fp32"] else torch.int32),
                           o2.view(torch.int16 if not d["out_fp32"] else torch.int32))


def test_report(cuda, capsys):
    with capsys.disabled():
        print("\n" + gemm_cases.report(f"production GEMM classes: {len(CASES)} distinct; per configuration: {COUNTS}; "
                                       f"wall time {time.time() - T0:.0f} s"))
