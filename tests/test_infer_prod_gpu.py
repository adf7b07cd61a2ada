"""Every distinct GEMM and glue launch of the two inference paths - the VAE and the few-step sampler - on the
GPU against float64.

tests/golden/infer_specs.json.gz holds one pointer-free spec per launch class of the recorded VAE encodes and
decodes (SD1.5 at 512^2, batches 8, 16 and 17; the SDXL config at 1024^2; a 264 x 256 image whose mid-block has
1056 tokens) and sampler calls (SD1.5 at guidance 1 and 7.5, SDXL, SD1.5 decoding inside the loop);
test_infer_specs_cpu.py keeps it equal to the plans.  Every class the training fixtures (gemm_specs.json.gz,
op_specs.json.gz, run by test_gemm_prod_gpu.py / test_op_prod_gpu.py) do not already hold runs here, exactly
as recorded, on NaN-poisoned buffers: GEMMs against gemm_spec.reference under gemm_spec.bound (a K-blocked
weight also re-run from row-major copies, bit for bit), ops against op_spec.reference under their derived
bounds.  Every byte outside the output windows must be unchanged.

The largest launches have 2^30 output elements: their references and checks run over slices of output
rows (each slice its own mean test), so the float64 copies of the whole result are never held at once."""
import ctypes
import os
import time

import pytest
import torch

import gemm_cases
import gemm_spec as G
import op_spec as O

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_INFER = O.trace.load(os.path.join(_HERE, "infer_specs.json.gz"))
_TRAIN_GEMM = {G.launch_class(s) for specs in G.trace.load(os.path.join(_HERE, "gemm_specs.json.gz")).values() for s in specs}
_TRAIN_OPS = {O.launch_class(s) for specs in O.trace.load(os.path.join(_HERE, "op_specs.json.gz")).values() for s in specs}

GEMMS, OPS, COUNTS = {}, {}, {}
for _name, _d in _INFER.items():
    for _i, _s in enumerate(_d["gemm"]):
        _k = G.launch_class(_s)
        if _k not in _TRAIN_GEMM:
            GEMMS.setdefault(_k, (f"{_name}-{_i}", _s))
    for _i, _s in enumerate(_d["ops"]):
        _k = O.launch_class(_s)
        if _k not in _TRAIN_OPS:
            OPS.setdefault(_k, (f"{_name}-{_i}-{_s['op'][4:]}", _s))
    COUNTS[_name] = (f"{len(_d['gemm'])} GEMM ({sum(G.launch_class(s) not in _TRAIN_GEMM for s in _d['gemm'])} new), "
                     f"{len(_d['ops'])} op ({sum(O.launch_class(s) not in _TRAIN_OPS for s in _d['ops'])} new)")
GEMM_CASES, OP_CASES = list(GEMMS.values()), list(OPS.values())
SLICE = 1 << 24            # output elements per float64 reference slice of a large GEMM
WORST, MARGIN, PEAK = {}, {}, [0]     # op family -> err / bound; GEMM family -> gemm_cases margin; bytes
T0 = time.time()


def _peak(fn):
    torch.cuda.reset_peak_memory_stats()
    fn()
    PEAK[0] = max(PEAK[0], torch.cuda.max_memory_allocated())


# ---------------------------------------------------------------------------------------------
# GEMMs
# ---------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _rowmajor_rerun(spec, T):
    """Launch again with every K-blocked weight replaced by a row-major copy of the same matrix."""
    from pcm_b200 import _lib
    d = spec["desc"]
    rows = {i: T.bsrc(b).contiguous() for i, b in enumerate(d["b"]) if b["kblocked"]}
    s = G.gemm_desc(d, T)
    for i, w in rows.items():
        s.b[i].ptr, s.b[i].ld, s.b[i].kblocked = w.data_ptr(), w.shape[1], 0
    _lib.check(_lib.lib().pcm_gemm(ctypes.byref(s), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pcm_gemm")
    torch.cuda.synchronize()


def _large(spec):
    return spec["desc"]["M"] * spec["desc"]["N"] > 4 * SLICE


def _sliced_run_and_check(spec, T, before):
    """gemm_cases.run_and_check over slices of output rows: launch, then per slice the float64 reference
    and gemm_spec.check (elementwise bound and mean test); then the guards, one buffer at a time.  Returns
    the destination window (a copy)."""
    d = spec["desc"]
    assert "pre" not in spec and d["residual"] != d["out"] and G.resolved_ksplit(d) == 1, \
        "a large launch reads only its inputs and writes only its destination"
    G.launch(spec, T)
    torch.cuda.synchronize()
    flat = T.flat(d["out"], torch.float32 if d["out_fp32"] else BF16)
    off, _ = G._row_offsets(d["M"], d["epiW"], d["epiHW"], d["osW"], d["osH"], d["osB"])
    off, cols = off.to(T.device), torch.arange(d["N"], device=T.device)
    out = torch.empty(d["M"], d["N"], dtype=flat.dtype, device=T.device)
    rows = max(1, SLICE // d["N"])
    worst = 0.0
    for m0 in range(0, d["M"], rows):
        m1 = min(d["M"], m0 + rows)
        out[m0:m1] = flat[off[m0:m1, None] + cols[None]]
        ref, S, base = G.reference(spec, T, rows=(m0, m1))
        worst = max(worst, G.check(out[m0:m1], ref, S, spec, base=base))
        del ref, S, base
    es = flat.element_size()
    lab = d["out"][0]
    for i, (b, b0) in enumerate(zip(T.bufs, before)):
        changed = b != b0
        if i == lab:
            for m0 in range(0, d["M"], rows):
                m1 = min(d["M"], m0 + rows)
                i16 = ((off[m0:m1, None] + cols[None]) * (es // 2) + d["out"][1] // 2).reshape(-1)
                changed[i16] = False
                if es == 4:
                    changed[i16 + 1] = False
        assert not changed.any(), f"buffer {i}: {int(changed.sum())} 2-byte words outside the destination window changed"
        del changed
    fam, steps = G.family(spec), sum(G.k_steps(spec))
    w0, s0 = MARGIN.get(fam, (0.0, 0))
    MARGIN[fam] = (max(w0, worst), max(s0, steps))
    return out


@pytest.mark.parametrize("spec", [c[1] for c in GEMM_CASES], ids=[c[0] for c in GEMM_CASES])
def test_inference_gemm(cuda, spec):
    saved, gemm_cases.MARGIN = gemm_cases.MARGIN, MARGIN       # this file's margins, apart from other modules'
    try:
        _peak(lambda: _gemm(cuda, spec))
    finally:
        gemm_cases.MARGIN = saved


def _gemm(cuda, spec):
    assert spec["op"] == "gemm" and "pre" not in spec
    d = spec["desc"]
    T = G.materialise(spec, cuda, seed=len(spec["spans"]))
    before = G.snapshot(T)
    if _large(spec):
        o1 = _sliced_run_and_check(spec, T, before)
    else:
        o1 = gemm_cases.run_and_check(spec, T, before)
    if G.resolved_ksplit(d) > 1:             # bit-reproducible: the slices are added in split order
        gemm_cases.restore(T, before)
        T.ws.fill_(float("nan"))
        G.launch(spec, T)
        torch.cuda.synchronize()
        assert torch.equal(_bits(o1), _bits(gemm_cases.result(spec, T)))
    if any(b["kblocked"] for b in d["b"]):   # K-blocked storage is a pure re-layout: bit-identical output
        gemm_cases.restore(T, before)
        del before
        _rowmajor_rerun(spec, T)
        flat = T.flat(d["out"], o1.dtype)
        off, _ = G._row_offsets(d["M"], d["epiW"], d["epiHW"], d["osW"], d["osH"], d["osB"])
        off, cols = off.to(cuda), torch.arange(d["N"], device=cuda)
        rows = max(1, SLICE // d["N"])
        for m0 in range(0, d["M"], rows):
            o2 = flat[off[m0:m0 + rows, None] + cols[None]]
            assert torch.equal(_bits(o1[m0:m0 + rows]), _bits(o2)), f"rows {m0}..: row-major weights give other bits"


# ---------------------------------------------------------------------------------------------
# glue and normalisation ops
# ---------------------------------------------------------------------------------------------
def _op_outputs(spec, T):
    return [T.bufs[lab][off // 2:(off + n + 1) // 2].clone() for lab, off, n in O.out_windows(spec)]


@pytest.mark.parametrize("spec", [c[1] for c in OP_CASES], ids=[c[0] for c in OP_CASES])
def test_inference_op(cuda, spec):
    _peak(lambda: _op(cuda, spec))


def _op(cuda, spec):
    T = O.materialise(spec, cuda, seed=len(spec["spans"]))
    before = T.snapshot()
    rc = O.launch(spec, T)
    assert rc == 0, _lib().pcm_last_error().decode()
    torch.cuda.synchronize()
    for k, v in O.check(spec, before, T).items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    O.guards(spec, T, before)
    if spec["op"] in O.GN_OPS:
        assert not T.ws[:4 * 3 * O.GN_MAX_B].any(), "the GroupNorm kernels must leave all three counter arrays at zero"
        o1 = _op_outputs(spec, T)            # fixed reduction order: a second launch gives the same bits
        for b, b0 in zip(T.bufs, before.bufs):
            b.copy_(b0)
        assert O.launch(spec, T) == 0
        torch.cuda.synchronize()
        for a, b in zip(o1, _op_outputs(spec, T)):
            assert torch.equal(a, b), f"{spec['op']}: a second launch on the same inputs differs"


def _lib():
    from pcm_b200 import _lib
    return _lib.lib()


def test_report(cuda, capsys):
    with capsys.disabled():
        per = "; ".join(f"{k}: {v}" for k, v in COUNTS.items())
        fam = ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items()))
        saved, gemm_cases.MARGIN = gemm_cases.MARGIN, MARGIN
        try:
            print("\n" + gemm_cases.report(
                f"inference launch classes run: {len(GEMM_CASES)} GEMM, {len(OP_CASES)} op (not in the training "
                f"fixtures); per configuration: {per}"))
        finally:
            gemm_cases.MARGIN = saved
        print(f"op families, largest err / bound: {fam}")
        print(f"device memory peak of one launch test: {PEAK[0] / 2 ** 30:.1f} GiB; "
              f"wall time {time.time() - T0:.0f} s (since the module was collected)")
