"""Pointer-free launch specs of the normalisation, glue and optimiser kernels (csrc/norm.cu, elementwise.cu,
optim.cu, and the VAE's glue in vae.cu), a float64 reference for each and a derived elementwise error bound.  Test infrastructure: nothing
under pcm_b200/ imports it.

A spec is plain data: the op name, its arguments as `ops._call` passed them (scalars as they are, pointers as
[buffer label, byte offset] with the labels renumbered per launch, None for an absent pointer) and `spans`,
the bytes of every buffer the launch's views cover, from the semantics in include/pcm_b200.h.  A GroupNorm
spec also carries `ws_bytes` (the dry run allocates no workspace), a `pcm_lora_refresh` spec its table.

`materialise` turns a spec into NaN-poisoned buffers with realistic values inside the input windows,
`launch` runs it through the C ABI with exactly the recorded scalars, `check` compares every output window
with `reference` under `bound`, and `guards` proves nothing outside the output windows changed.  The
reference runs on any torch device, so the checker itself is tested on the CPU (tests/test_op_specs_cpu.py).
"""
import contextlib
import copy
import ctypes
import functools
import json
import math

import torch

from gemm_spec import NUM_SMS, POISON, TAIL, trace  # noqa: F401  (trace: the launch recorder)

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24             # fp32 unit roundoff (round to nearest, 24-bit significand)
U_FAST = 2.0 ** -22        # relative error of __expf / frcp_approx / rsqrtf / erff (a few fp32 ulps)

# argument names of every covered op, in C ABI order without the trailing stream
ARGS = {
    "pcm_groupnorm_fwd": "x1 x2 C1 C2 B HW G gamma beta eps silu out stats ws ws_bytes",
    "pcm_groupnorm_fwd_part": "x1 x2 C1 C2 B part_B HW G gamma beta eps silu out stats ws ws_bytes",
    "pcm_groupnorm_bwd": "dy x1 x2 C1 C2 B HW G gamma beta eps silu stats red add dx1 dx2 colsum ws ws_bytes",
    "pcm_layernorm_fwd": "x M C gamma beta eps out stats",
    "pcm_layernorm_bwd": "dy x M C gamma stats add dx",
    "pcm_geglu_fwd": "u M F out",
    "pcm_geglu_bwd": "dgg u M F du",
    "pcm_upsample2x_fwd": "x B H W C out",
    "pcm_upsample2x_bwd": "dout B H W C din",
    "pcm_conv3x3_c4": "x B H W C w bias sgn round_in out",
    "pcm_timestep_embed": "t B C out",
    "pcm_add_bf16": "a b n out",
    "pcm_cast_f32_bf16": "x n out",
    "pcm_grad_sumsq": "g n out",
    "pcm_adamw_clip": "p g m v n state beta1 beta2 eps wd max_norm inv_world sumsq zero_grad",
    "pcm_ema_update": "targ src n rate",
    "pcm_lora_refresh": "master table num_entries total_work scale opnd",
    "pcm_softmax_rows": "s rows cols lds p ldp",
    "pcm_transpose_bf16": "in rows cols ldi bsi batch out ldo bso",
    "pcm_latent_dist": "h B HW w bias noise scale mean logvar std sample",
    "pcm_vae_dec_in": "z M w bias div out",
    "pcm_image_exit": "x B HW C out u8",
}
ARGS = {k: v.split() for k, v in ARGS.items()}
# `_call` entry points with suites of their own: attention (test_attn_*), the PCM solver arithmetic
# (test_pcm_kernels_gpu against the pinned oracle) and the sampler's LoRA fuse / DDIM step (test_sampler_gpu);
# pcm_colsum is no launch of the training step (GroupNorm's backward sums the time-embedding gradient)
OUT_OF_SCOPE = {"pcm_attn_fwd", "pcm_attn_bwd", "pcm_prepare", "pcm_add_noise", "pcm_teacher_step",
                "pcm_teacher_substep", "pcm_loss", "pcm_noise_travel", "pcm_axpby_f64", "pcm_fm_step",
                "pcm_sample_step", "pcm_lora_fuse", "pcm_colsum"}
GN_OPS = ("pcm_groupnorm_fwd", "pcm_groupnorm_fwd_part", "pcm_groupnorm_bwd")
# the pointers a launch only reads / writes (a pointer in both is updated in place)
_OUTS = {
    "pcm_groupnorm_fwd": ("out", "stats"), "pcm_groupnorm_fwd_part": ("out", "stats"),
    "pcm_groupnorm_bwd": ("red", "dx1", "dx2", "colsum"), "pcm_layernorm_fwd": ("out", "stats"),
    "pcm_layernorm_bwd": ("dx",), "pcm_geglu_fwd": ("out",), "pcm_geglu_bwd": ("du",),
    "pcm_upsample2x_fwd": ("out",), "pcm_upsample2x_bwd": ("din",), "pcm_conv3x3_c4": ("out",),
    "pcm_timestep_embed": ("out",), "pcm_add_bf16": ("out",), "pcm_cast_f32_bf16": ("out",),
    "pcm_grad_sumsq": ("out",), "pcm_adamw_clip": ("p", "g", "m", "v", "state"), "pcm_ema_update": ("targ",),
    "pcm_lora_refresh": ("opnd",), "pcm_softmax_rows": ("p",), "pcm_transpose_bf16": ("out",),
    "pcm_latent_dist": ("mean", "logvar", "std", "sample"), "pcm_vae_dec_in": ("out",),
    "pcm_image_exit": ("out", "u8"),
}
SUMSQ_WS_DOUBLES = 1024


# ---------------------------------------------------------------------------------------------
# launch configurations restated from the kernels' host code (132 SMs: the H100 SXM of the recorded plans)
# ---------------------------------------------------------------------------------------------
GN_MAX_C, GN_STAGE, GN_MAX_B = 2560, 4096, 1024


def gn_launch_cfg(C, HW, B, sms=NUM_SMS):
    """(threads, pixels per block, blocks per image) of csrc/norm.cu gn_launch_cfg; None where it rejects C."""
    nvec = C // 8
    if C % 8 or C > GN_MAX_C or nvec > 1024:
        return None
    ny = max(1, 512 // nvec)
    target = max(1, (2 * sms) // B)
    p = max(-(-HW // target), ny * 4)
    if -(-HW // p) > 128:
        p = -(-HW // 128)
    return nvec * ny, p, -(-HW // p)


def gn_ws_need(B, nblk, C, G):
    return 4 * 3 * GN_MAX_B + 4 * B * nblk * (2 * G + C)


def gn_ws_bytes(B, HW, C, G):
    """pcm_groupnorm_ws_bytes: the need of a single-image partition (an upper bound for any batch)."""
    cfg = gn_launch_cfg(C, HW, 1)
    return -1 if cfg is None else gn_ws_need(B, cfg[2], C, G)


def sumsq_grid(n, sms=NUM_SMS):
    return max(1, min(-(-(n // 4) // 256), 4 * sms, SUMSQ_WS_DOUBLES - 2))


# ---------------------------------------------------------------------------------------------
# spec_of / launch_class / distinct_specs
# ---------------------------------------------------------------------------------------------
def _refresh_rows(table):
    for a_off, b_off, a_fwd, sb_fwd, sb_t, a_t, ci, co, w0 in table:
        yield dict(a_off=a_off, b_off=b_off, a_fwd=a_fwd, sb_fwd=sb_fwd, sb_t=sb_t, a_t=a_t,
                   cin=ci & 0xFFFFFFFF, taps=ci >> 32, n=co & 0xFFFFFFFF, r=co >> 32, work=w0)


def extents(op, a, table=None):
    """{pointer name: bytes its view covers} of one launch, from the op's semantics."""
    if op in GN_OPS:
        C = a["C1"] + a["C2"]
        px = a["B"] * a["HW"]
        e = dict(x1=2 * px * a["C1"], x2=2 * px * a["C2"], gamma=4 * C, beta=4 * C, stats=8 * a["B"] * a["G"])
        if op == "pcm_groupnorm_bwd":
            e.update(dy=2 * px * C, add=2 * px * C, dx1=2 * px * a["C1"], dx2=2 * px * a["C2"],
                     red=8 * a["B"] * a["G"], colsum=4 * a["B"] * C)
        else:
            e.update(out=2 * px * C)
        return e
    if op == "pcm_layernorm_fwd":
        return dict(x=2 * a["M"] * a["C"], gamma=4 * a["C"], beta=4 * a["C"], out=2 * a["M"] * a["C"], stats=8 * a["M"])
    if op == "pcm_layernorm_bwd":
        n = 2 * a["M"] * a["C"]
        return dict(dy=n, x=n, gamma=4 * a["C"], stats=8 * a["M"], add=n, dx=n)
    if op == "pcm_geglu_fwd":
        return dict(u=4 * a["M"] * a["F"], out=2 * a["M"] * a["F"])
    if op == "pcm_geglu_bwd":
        return dict(dgg=2 * a["M"] * a["F"], u=4 * a["M"] * a["F"], du=4 * a["M"] * a["F"])
    if op.startswith("pcm_upsample2x"):
        n = 2 * a["B"] * a["H"] * a["W"] * a["C"]
        return dict(x=n, out=4 * n) if op.endswith("fwd") else dict(dout=4 * n, din=n)
    if op == "pcm_conv3x3_c4":
        px = a["B"] * a["H"] * a["W"]
        return dict(x=16 * px, w=72 * a["C"], bias=4 * a["C"], out=2 * px * a["C"])
    if op == "pcm_timestep_embed":
        return dict(t=8 * a["B"], out=2 * a["B"] * a["C"])
    if op == "pcm_add_bf16":
        return dict(a=2 * a["n"], b=2 * a["n"], out=2 * a["n"])
    if op == "pcm_cast_f32_bf16":
        return dict(x=4 * a["n"], out=2 * a["n"])
    if op == "pcm_grad_sumsq":
        return dict(g=4 * a["n"], out=8 * SUMSQ_WS_DOUBLES)
    if op == "pcm_adamw_clip":
        n = 4 * a["n"]
        return dict(p=n, g=n, m=n, v=n, state=8, sumsq=8)
    if op == "pcm_ema_update":
        return dict(targ=4 * a["n"], src=4 * a["n"])
    if op == "pcm_lora_refresh":
        rows = list(_refresh_rows(table))
        master = max(max(e["a_off"] + e["r"] * e["taps"] * e["cin"], e["b_off"] + e["n"] * e["r"]) for e in rows)
        opnd = max(max(e["a_fwd"], e["a_t"]) + e["r"] * e["taps"] * e["cin"] for e in rows)
        opnd = max(opnd, max(max(e["sb_fwd"], e["sb_t"]) + e["n"] * e["r"] for e in rows))
        return dict(master=4 * master, table=72 * a["num_entries"], opnd=2 * opnd)
    if op == "pcm_softmax_rows":
        return dict(s=4 * ((a["rows"] - 1) * a["lds"] + a["cols"]), p=2 * ((a["rows"] - 1) * a["ldp"] + a["cols"]))
    if op == "pcm_transpose_bf16":
        return {"in": 2 * ((a["batch"] - 1) * a["bsi"] + (a["rows"] - 1) * a["ldi"] + a["cols"]),
                "out": 2 * ((a["batch"] - 1) * a["bso"] + (a["cols"] - 1) * a["ldo"] + a["rows"])}
    if op == "pcm_latent_dist":
        n = 16 * a["B"] * a["HW"]
        return dict(h=2 * n, w=2 * 64, bias=4 * 8, noise=n, mean=n, logvar=n, std=n, sample=n)
    if op == "pcm_vae_dec_in":
        return dict(z=16 * a["M"], w=2 * 16, bias=4 * 4, out=16 * a["M"])
    if op == "pcm_image_exit":
        n = a["B"] * a["HW"] * a["C"]
        return dict(x=4 * n, out=4 * n, u8=n)
    raise KeyError(op)


def make_spec(op, refresh_table=None, **args):
    """A spec from named arguments; a pointer is a [label, offset] list, or True for a buffer of its own
    (`refresh_table`: the rows of a `pcm_lora_refresh` table)."""
    a, n = {}, 0
    ptrs = set(extents(op, args, refresh_table)) | {"ws"}
    for k in ARGS[op]:
        v = args.get(k)
        assert k not in ptrs or v is None or v is True or isinstance(v, list), f"{op}: pointer {k} = {v!r}"
        if v is True:
            v = [n, 0]
            n += 1
        a[k] = v
    return _finish(op, a, refresh_table)


def _finish(op, a, table):
    spec = dict(op=op, args=a)
    if table is not None:
        spec["table"] = table
    labels, spans = {}, {}
    for k in ARGS[op]:
        if isinstance(a[k], list):
            a[k][0] = labels.setdefault(a[k][0], len(labels))
    for k, nbytes in extents(op, a, table).items():
        if isinstance(a.get(k), list):
            spans[a[k][0]] = max(spans.get(a[k][0], 0), a[k][1] + nbytes)
    spec["spans"] = [spans[i] for i in range(len(labels))]
    if op in GN_OPS:
        a["ws"], a["ws_bytes"] = None, 0
        spec["ws_bytes"] = gn_ws_bytes(a["B"], a["HW"], a["C1"] + a["C2"], a["G"])
    return spec


def spec_of(rec):
    """One recorded `ops._call` launch (a trace record with op / args [/ table]) as a spec."""
    op = rec["op"]
    a = dict(zip(ARGS[op], copy.deepcopy(rec["args"])))
    assert len(a) == len(rec["args"]), (op, rec["args"])
    return _finish(op, a, copy.deepcopy(rec.get("table")))


def launch_class(spec):
    """The op, its scalars, which pointers are absent and which share a buffer: the byte offsets inside
    the buffers are dropped (another window of the same buffers runs the same instructions)."""
    a = {k: (v[0] if isinstance(v, list) else v) for k, v in spec["args"].items()}
    key = dict(op=spec["op"], args=a, table=spec.get("table"))
    return json.dumps(key, sort_keys=True, separators=(",", ":"))


def distinct_specs(records):
    """The first spec of every launch class among the covered ops of a recorded trace, in launch order."""
    seen, out = set(), []
    for r in records:
        if r["op"] in ARGS:
            s = spec_of(r)
            k = launch_class(s)
            if k not in seen:
                seen.add(k)
                out.append(s)
    return out


def family(spec):
    op = spec["op"][4:]
    a = spec["args"]
    if spec["op"] in GN_OPS:
        return op + ("" if a["x2"] is None else " concat") + (" +colsum" if a.get("colsum") else "")
    return op


@contextlib.contextmanager
def recording():
    """Record one dry-run step (nothing launches): yields the Recorder of make_launch_trace.py, whose trace
    additionally holds the table contents of every `pcm_lora_refresh` (read while the table is alive)."""
    import pytest
    from pcm_b200 import ops
    rec = trace.Recorder()
    with pytest.MonkeyPatch.context() as mp:
        trace._install(mp, rec)
        call = ops._call

        def rec_call(name, *args):
            call(name, *args)
            if name == "pcm_lora_refresh":
                flat = list((ctypes.c_int64 * (9 * args[2])).from_address(args[1]))
                rec.trace[-1]["table"] = [flat[9 * i:9 * i + 9] for i in range(args[2])]

        mp.setattr(ops, "_call", rec_call)
        yield rec


# ---------------------------------------------------------------------------------------------
# materialise
# ---------------------------------------------------------------------------------------------
class Tensors:
    """The buffers of a materialised spec: `bufs[label]` is an int16 tensor (span + TAIL, rounded to 16
    bytes), the NaN pattern wherever nothing was written."""

    def __init__(self, spec, device, bufs=None):
        self.spec, self.device = spec, device
        self.bufs = bufs if bufs is not None else [
            torch.full(((n + 15) // 16 * 8 + TAIL // 2,), POISON, dtype=torch.int16, device=device) for n in spec["spans"]]
        self.ws = None

    def view(self, name, dtype, n=None):
        """1-D typed view of pointer `name`: from its byte offset, `n` elements (default: to the span)."""
        p = self.spec["args"][name]
        if p is None:
            return None
        b = self.bufs[p[0]].view(torch.uint8)[p[1]:]
        es = torch.tensor([], dtype=dtype).element_size()
        if n is None:
            n = (self.spec["spans"][p[0]] - p[1]) // es
        return b[:n * es].view(dtype)

    def addr(self, name):
        p = self.spec["args"][name]
        return 0 if p is None else self.bufs[p[0]].data_ptr() + p[1]

    def snapshot(self):
        return Tensors(self.spec, self.device, [b.clone() for b in self.bufs])


def _g(gen, n, scale=1.0, mean=0.0):
    return torch.randn(n, generator=gen, device=gen.device, dtype=F32) * scale + mean


def _channels(gen, npix, C, outliers=True):
    """[npix, C] activations like a pretrained UNet's: unit-scale noise, every 16th channel (from channel 5)
    with a per-channel mean of 20 - 60 sigma."""
    x = _g(gen, npix * C).view(npix, C)
    if outliers:
        off = torch.zeros(C, device=gen.device)
        off[5::16] = (20 + 40 * torch.rand(len(off[5::16]), generator=gen, device=gen.device)) * \
            torch.sign(torch.randn(len(off[5::16]), generator=gen, device=gen.device))
        x += off
    return x


def _affine(gen, C):
    gamma, beta = _g(gen, C, 0.2, 1.0), _g(gen, C, 0.2)
    gamma[3::29] = 0.0                     # the gm != 0 branch of gn_bwd_stats_kernel
    return gamma, beta


def materialise(spec, device, seed=0):
    """Every buffer poisoned, then seeded realistic values inside each input window; outputs stay NaN
    (a pointer that is both read and written - AdamW's state, EMA's target - holds input values)."""
    T = Tensors(spec, device)
    g = torch.Generator(device=device).manual_seed(seed)
    op, a = spec["op"], spec["args"]
    if op in GN_OPS:
        C1, C2, B, HW = a["C1"], a["C2"], a["B"], a["HW"]
        x = _channels(g, B * HW, C1 + C2).to(BF16)
        T.view("x1", BF16, B * HW * C1).view(B * HW, C1).copy_(x[:, :C1])
        if C2:
            T.view("x2", BF16, B * HW * C2).view(B * HW, C2).copy_(x[:, C1:])
        gamma, beta = _affine(g, C1 + C2)
        T.view("gamma", F32, C1 + C2).copy_(gamma)
        T.view("beta", F32, C1 + C2).copy_(beta)
        if op == "pcm_groupnorm_bwd":
            T.view("dy", BF16, B * HW * (C1 + C2)).copy_(_g(g, B * HW * (C1 + C2), 0.05).to(BF16))
            if a["add"]:
                T.view("add", BF16, B * HW * (C1 + C2)).copy_(_g(g, B * HW * (C1 + C2), 0.05).to(BF16))
            if (C1 + C2) % a["G"] == 0:      # (a launch the host code rejects has no statistics)
                T.view("stats", F32, 2 * B * a["G"]).copy_(gn_stats64(T, a["eps"]).reshape(-1).float())
        T.ws = torch.zeros(max(spec["ws_bytes"], 0), dtype=torch.uint8, device=device)
    elif op == "pcm_layernorm_fwd" or op == "pcm_layernorm_bwd":
        M, C = a["M"], a["C"]
        T.view("x", BF16, M * C).copy_(_channels(g, M, C, outliers=False).reshape(-1).to(BF16))
        gamma, beta = _affine(g, C)
        T.view("gamma", F32, C).copy_(gamma)
        if op == "pcm_layernorm_fwd":
            T.view("beta", F32, C).copy_(beta)
        else:
            T.view("dy", BF16, M * C).copy_(_g(g, M * C, 0.05).to(BF16))
            if a["add"]:
                T.view("add", BF16, M * C).copy_(_g(g, M * C, 0.05).to(BF16))
            x = T.view("x", BF16, M * C).view(M, C).double()
            m = x.mean(1)
            r = ((x - m[:, None]).pow(2).mean(1) + float(torch.tensor(1e-5, dtype=F32))).rsqrt()
            T.view("stats", F32, 2 * M).copy_(torch.stack([m, r], 1).reshape(-1).float())
    elif op in ("pcm_geglu_fwd", "pcm_geglu_bwd"):
        M, Fh = a["M"], a["F"]
        T.view("u", BF16, 2 * M * Fh).copy_(_g(g, 2 * M * Fh, 1.5).to(BF16))
        if op == "pcm_geglu_bwd":
            T.view("dgg", BF16, M * Fh).copy_(_g(g, M * Fh, 0.05).to(BF16))
    elif op.startswith("pcm_upsample2x"):
        n = a["B"] * a["H"] * a["W"] * a["C"]
        if op.endswith("fwd"):
            T.view("x", BF16, n).copy_(_g(g, n).to(BF16))
        else:
            T.view("dout", BF16, 4 * n).copy_(_g(g, 4 * n).to(BF16))
    elif op == "pcm_conv3x3_c4":
        n, C = a["B"] * a["H"] * a["W"], a["C"]
        T.view("x", F32, 4 * n).copy_(_g(g, 4 * n))
        T.view("w", BF16, 36 * C).copy_(_g(g, 36 * C, 0.2).to(BF16))
        if a["bias"]:
            T.view("bias", F32, C).copy_(_g(g, C, 0.2))
    elif op == "pcm_timestep_embed":
        T.view("t", torch.int64, a["B"]).copy_(torch.randint(0, 1000, (a["B"],), generator=g, device=device))
    elif op == "pcm_add_bf16":
        T.view("a", BF16, a["n"]).copy_(_g(g, a["n"]).to(BF16))
        T.view("b", BF16, a["n"]).copy_(_g(g, a["n"]).to(BF16))
    elif op == "pcm_cast_f32_bf16":
        T.view("x", F32, a["n"]).copy_(_g(g, a["n"]))
    elif op == "pcm_grad_sumsq":
        T.view("g", F32, a["n"]).copy_(_g(g, a["n"], 1e-3))
        T.view("out", F64, SUMSQ_WS_DOUBLES).zero_()
    elif op == "pcm_adamw_clip":
        n = a["n"]
        T.view("p", F32, n).copy_(_g(g, n, 0.02))
        T.view("g", F32, n).copy_(_g(g, n, 1e-3))
        T.view("m", F32, n).copy_(_g(g, n, 1e-4))
        T.view("v", F32, n).copy_(_g(g, n, 1e-4).square())
        T.view("state", F32, 2).copy_(torch.tensor([1e-4, 0.0], device=device))
        T.view("sumsq", F64, 1).fill_(sumsq64(T.view("g", F32, n)))
    elif op == "pcm_ema_update":
        T.view("targ", F32, a["n"]).copy_(_g(g, a["n"], 0.02))
        T.view("src", F32, a["n"]).copy_(_g(g, a["n"], 0.02))
    elif op == "pcm_lora_refresh":
        T.view("master", F32).copy_(_g(g, T.view("master", F32).numel(), 0.05))
        T.view("table", torch.int64, 9 * a["num_entries"]).copy_(torch.tensor(spec["table"], device=device).view(-1))
    elif op == "pcm_softmax_rows":
        rows, cols = a["rows"], a["cols"]
        # attention scores: each row N(0, sigma^2), sigma from 0.5 (flat) to 6 (peaked); the last row shifted
        # by +90, where exp without the max subtraction overflows fp32
        sig = 0.5 + 5.5 * torch.rand(rows, 1, generator=g, device=device)
        s, step = softmax_scores(T), max(1, (1 << 24) // cols)
        for r0 in range(0, rows, step):
            r1 = min(rows, r0 + step)
            s[r0:r1] = _g(g, (r1 - r0) * cols).view(r1 - r0, cols) * sig[r0:r1]
        s[rows - 1] += 90.0
    elif op == "pcm_transpose_bf16":
        v = transpose_views(T)[0]
        v.copy_(_g(g, v.numel()).view(v.shape).to(BF16))
    elif op == "pcm_latent_dist":
        n = a["B"] * a["HW"]
        # encoder.conv_out pixels, not bf16 values (the kernel rounds its inputs); every 7th pixel 40 times
        # larger, so moments land past both logvar clamps
        h = _g(g, 8 * n, 2.0).view(n, 8)
        h[::7] *= 40.0
        T.view("h", F32, 8 * n).copy_(h.view(-1))
        T.view("w", BF16, 64).copy_(_g(g, 64, 0.35).to(BF16))
        T.view("bias", F32, 8).copy_(_g(g, 8, 0.5))
        if a["noise"]:
            T.view("noise", F32, 4 * n).copy_(_g(g, 4 * n))
    elif op == "pcm_vae_dec_in":
        M = a["M"]
        T.view("z", F32, 4 * M).copy_(_g(g, 4 * M))
        T.view("w", BF16, 16).copy_(_g(g, 16, 0.5).to(BF16))
        T.view("bias", F32, 4).copy_(_g(g, 4, 0.1))
    elif op == "pcm_image_exit":
        n = a["B"] * a["HW"] * a["C"]
        x = T.view("x", F32, n)
        x.copy_(_g(g, n, 0.7))                      # |x| > 1 (clamped) in 15 per cent of the values
        ties = image_exit_ties().to(device)
        k = min(n, len(ties))
        x[:k] = ties[:k]                            # v * 255 exactly k + 1/2 (round half to even) ...
        x[n - k:] = ties[:k].flip(0)                # ... in the first and the last image
    else:
        raise KeyError(op)
    return T


def softmax_scores(T):
    """[rows, cols] fp32 view of a pcm_softmax_rows spec's scores (row stride lds)."""
    a = T.spec["args"]
    return T.view("s", F32).as_strided((a["rows"], a["cols"]), (a["lds"], 1))


def transpose_views(T):
    """(input [batch, rows, cols], output [batch, cols, rows]) bf16 views of a pcm_transpose_bf16 spec."""
    a = T.spec["args"]
    return (T.view("in", BF16).as_strided((a["batch"], a["rows"], a["cols"]), (a["bsi"], a["ldi"], 1)),
            T.view("out", BF16).as_strided((a["batch"], a["cols"], a["rows"]), (a["bso"], a["ldo"], 1)))


@functools.lru_cache(None)
def image_exit_ties():
    """fp32 inputs x whose image value v = x / 2 + 0.5 (fp32) makes v * 255 (fp32) exactly k + 1/2, for
    every k in [0, 255) that has one: the ties round(v * 255) rounds to even."""
    out = []
    for k in range(255):
        b0 = int(torch.tensor([(k + 0.5) / 255], dtype=F32).view(torch.int32))
        for b in range(b0 - 8, b0 + 9):                 # the fp32 values within 8 ulps
            v = torch.tensor([b], dtype=torch.int32).view(F32)
            x = ((v.double() - 0.5) * 2).float()
            if float(v * 255) == k + 0.5 and torch.equal(x / 2 + 0.5, v):
                out.append(float(x))
                break
    return torch.tensor(out, dtype=F32)


# ---------------------------------------------------------------------------------------------
# reference and bound
# ---------------------------------------------------------------------------------------------
def half_ulp_bf16(x):
    """Half a bf16 ulp at magnitude |x| (x float64): the largest error of one round-to-nearest to bf16.
    Zero and subnormal magnitudes get the subnormal spacing."""
    e = torch.frexp(x.abs().clamp_min(2.0 ** -126))[1] - 1     # |x| in [2^e, 2^(e+1))
    return torch.ldexp(torch.ones_like(x), e - 8)


def bf16_bound(ref, e):
    """One bf16 rounding of a value within e of ref: e + half an ulp of the largest value it can be."""
    return e + half_ulp_bf16(ref.abs() + e)


def f32(x):
    """A float argument as the kernel receives it (rounded to fp32), as a Python float."""
    return float(torch.tensor(x, dtype=F32))


class Piece:
    """One compared output window: `got` (the output, any dtype) against `ref` within `bnd` (or bit for bit
    when `bnd` is None).  `signed`: weights w for the mean signed error test (see `check`)."""

    def __init__(self, fam, got, ref, bnd=None, signed=None, e_fp32=None):
        self.fam, self.got, self.ref, self.bnd, self.signed, self.e_fp32 = fam, got, ref, bnd, signed, e_fp32


def _silu(y):
    return y * torch.sigmoid(y)


def _dsilu(y):
    s = torch.sigmoid(y)
    return s * (1 + y * (1 - s))


def gn_stats64(T, eps):
    """[B, G, 2] float64 (mean, rstd) of a GroupNorm spec's input; eps as the kernel receives it."""
    a = T.spec["args"]
    out = []
    for b in range(a["B"]):
        X = gn_image(T, b)
        Xg = X.view(a["HW"], a["G"], -1)
        m = Xg.mean((0, 2))
        v = (Xg - m[None, :, None]).square().mean((0, 2))
        out.append(torch.stack([m, (v + f32(eps)).rsqrt()], 1))
    return torch.stack(out)


def gn_image(T, b):
    """[HW, C] float64 input of image b (x1 | x2)."""
    a = T.spec["args"]
    HW, C1, C2 = a["HW"], a["C1"], a["C2"]
    x1 = T.view("x1", BF16, a["B"] * HW * C1).view(a["B"], HW, C1)[b].double()
    if not C2:
        return x1
    return torch.cat([x1, T.view("x2", BF16, a["B"] * HW * C2).view(a["B"], HW, C2)[b].double()], 1)


def gn_depth(a):
    """Summation depth of one group statistic in csrc/norm.cu: a thread's pixel loop, the ny staged rows,
    the channels of a group and the block partials (each a linear chain in the worst case)."""
    threads, ppb, nblk = gn_launch_cfg(a["C1"] + a["C2"], a["HW"], a.get("part_B", a["B"]))
    ny = threads // ((a["C1"] + a["C2"]) // 8)
    return -(-ppb // ny) + ny + (a["C1"] + a["C2"]) // a["G"] + nblk + 8


def gn_stats_bound(X, G, eps, depth):
    """(mean bound, rstd relative bound) [G] of the kernel's statistics of one image X [HW, C] float64.

    The kernel sums d = x - pivot per channel (pivot: the channel's value at pixel 0 of the image; bf16
    minus bf16 is exact in fp32), and d^2, in fp32 chains of at most `depth` additions: a sum is within
    depth * 2^-24 * sum|terms| of the exact one.  The channel means piv + s/n then have an error of
        dm <= depth * u * (mean|d| + mean|x|)
    and the channel M2 = sum d^2 - s^2/n (s^2/n <= sum d^2) one of (depth + 3) u sum d^2.  Chan's merges
    of channels and blocks add the between-part terms n (m_c - m)^2, each exact up to (depth) u of itself
    plus 2 n |m_c - m| dm.  With A2 = mean d^2 + mean (m_c - m)^2 + var over the group:
        dv <= (depth + 4) u A2 + 2 dm sqrt(A2) + dm^2,
    and rstd = rsqrt(v + eps) moves by half the relative error of v + eps, plus rsqrtf and roundings
    (6 u).  The pivot makes A2 ~ var when the data have no outlier at pixel 0 (the |mean| >> sigma of
    pretrained channels cancels exactly); an outlier pivot of k sigma raises A2 to ~ k^2 sigma^2, and the
    bound with it: the kernel's variance is only that accurate there."""
    HW, C = X.shape
    cpg = C // G
    d = X - X[0:1]
    Xg, dg = X.view(HW, G, cpg), d.view(HW, G, cpg)
    m = Xg.mean((0, 2))
    mc = X.mean(0).view(G, cpg)
    var = (Xg - m[None, :, None]).square().mean((0, 2))
    dm = depth * U * (dg.abs().mean((0, 2)) + Xg.abs().mean((0, 2)))
    A2 = dg.square().mean((0, 2)) + (mc - m[:, None]).square().mean(1) + var
    dv = (depth + 4) * U * A2 + 2 * dm * A2.sqrt() + dm * dm
    dr = 0.5 * (dv + 2 * U * var) / (var + f32(eps)) + 6 * U
    return dm, dr


def _gn_ref(spec, Tin, Tout):
    a = spec["args"]
    B, HW, G, C1, C2 = a["B"], a["HW"], a["G"], a["C1"], a["C2"]
    C, cpg, eps, silu = C1 + C2, (C1 + C2) // G, f32(a["eps"]), a["silu"]
    depth = gn_depth(a)
    gamma, beta = Tin.view("gamma", F32, C).double(), Tin.view("beta", F32, C).double()
    chan_g = torch.arange(C, device=gamma.device) // cpg
    if spec["op"] != "pcm_groupnorm_bwd":
        stats = Tout.view("stats", F32, 2 * B * G).view(B, G, 2)
        out = Tout.view("out", BF16, B * HW * C).view(B, HW, C)
        for b in range(B):
            X = gn_image(Tin, b)
            Xg = X.view(HW, G, cpg)
            m = Xg.mean((0, 2))
            r = ((Xg - m[None, :, None]).square().mean((0, 2)) + eps).rsqrt()
            dm, dr = gn_stats_bound(X, G, eps, depth)
            yield Piece("gn stats", stats[b, :, 0], m, dm)
            yield Piece("gn stats", stats[b, :, 1], r, dr * r)
            # the output against float64 arithmetic on the kernel's own statistics (checked just above):
            # x * sc + sh with sc = rstd * gamma, sh = beta - mean * sc in fp32, three roundings of the
            # largest of |x sc|, |mean sc|, |beta|; SiLU (slope <= 1.1, fast exp / reciprocal), one bf16 rounding
            mk, rk = stats[b, :, 0].double()[chan_g], stats[b, :, 1].double()[chan_g]
            sc = rk * gamma
            y = (X - mk) * sc + beta
            e = 3 * U * ((X * sc).abs() + (mk * sc).abs() + beta.abs())
            if silu:
                ref = _silu(y)
                e = 1.1 * e + U_FAST * (4 + y.abs()) * ref.abs()
            else:
                ref = y
            yield Piece("gn fwd", out[b], ref, bf16_bound(ref, e))
        return
    stats = Tin.view("stats", F32, 2 * B * G).view(B, G, 2).double()
    red = Tout.view("red", F32, 2 * B * G).view(B, G, 2)
    dx1 = Tout.view("dx1", BF16, B * HW * C1).view(B, HW, C1)
    dx2 = Tout.view("dx2", BF16, B * HW * C2).view(B, HW, C2) if C2 else None
    colsum = Tout.view("colsum", F32, B * C).view(B, C) if a["colsum"] else None
    dy_all = Tin.view("dy", BF16, B * HW * C).view(B, HW, C)
    add_all = Tin.view("add", BF16, B * HW * C).view(B, HW, C) if a["add"] else None
    n = HW * cpg
    inv_n = f32(1.0 / n)
    for b in range(B):
        X, dy = gn_image(Tin, b), dy_all[b].double()
        m, r = stats[b, :, 0][chan_g], stats[b, :, 1][chan_g]
        U_, V_ = r * gamma, beta - m * r * gamma
        pre = X * U_ + V_
        e_pre = 3 * U * ((X * U_).abs() + (m * U_).abs() + beta.abs())
        ds = _dsilu(pre) if silu else torch.ones_like(pre)
        # dsilu: |dsilu'| <= 0.5, fast sigmoid; without SiLU exact
        e_ds = (0.5 * e_pre + U_FAST * (4 + pre.abs())) if silu else torch.zeros_like(pre)
        gd = dy * gamma
        g = gd * ds
        xh = (X - m) * r
        # red = (sum g, sum g xhat), the second accumulated as sum g pre and converted by (q - beta a) / gamma
        s0 = g.view(HW, G, cpg).sum((0, 2))
        s1 = (g * xh).view(HW, G, cpg).sum((0, 2))
        e0c = depth * U * g.abs().sum(0) + (gd.abs() * e_ds).sum(0) + 2 * U * g.abs().sum(0)
        q_abs = (g * pre).abs().sum(0)
        e1c = depth * U * q_abs + (g.abs() * e_pre).sum(0) + (gd.abs() * e_ds * pre.abs()).sum(0) \
            + beta.abs() * e0c + 2 * U * (q_abs + (beta * g.sum(0)).abs())
        e1c = torch.where(gamma != 0, e1c / gamma.abs().clamp_min(1e-30), torch.zeros_like(e1c)) \
            + 2 * U * (g * xh).sum(0).abs()
        e0 = e0c.view(G, cpg).sum(1) + depth * U * g.abs().view(HW, G, cpg).sum((0, 2))
        e1 = e1c.view(G, cpg).sum(1) + depth * U * (g * xh).abs().view(HW, G, cpg).sum((0, 2))
        yield Piece("gn red", red[b, :, 0], s0, e0)
        yield Piece("gn red", red[b, :, 1], s1, e1)
        # dx on the kernel's own red (checked above): U dyh + x P + Q (+ add) in fp32
        k0 = red[b, :, 0].double()[chan_g] * inv_n
        k1 = red[b, :, 1].double()[chan_g] * inv_n
        ad = add_all[b].double() if add_all is not None else 0.0
        ref = r * (g - k0 - xh * k1) + ad
        P_, Q_ = -r * r * k1, -r * k0 + m * r * r * k1
        e = 3 * U * (U_ * dy * ds).abs() + (U_ * dy).abs() * e_ds + 4 * U * ((X * P_).abs() + (m * P_).abs()
                                                                          + (r * k0).abs() + (ref - ad).abs())
        if add_all is not None:
            e = e + 2 * U * (ref.abs() + ad.abs())
        bnd = bf16_bound(ref, e)
        yield Piece("gn bwd", dx1[b], ref[:, :C1], bnd[:, :C1])
        if C2:
            yield Piece("gn bwd", dx2[b], ref[:, C1:], bnd[:, C1:])
        if colsum is not None:
            # the fp32 values before their bf16 rounding, summed over the image in fp32 chains
            yield Piece("gn colsum", colsum[b], ref.sum(0), e.sum(0) + depth * U * ref.abs().sum(0))


def _ln_ref(spec, Tin, Tout, rows=8192):
    a = spec["args"]
    M, C = a["M"], a["C"]
    lpr = 8 if C // 8 <= 40 else (16 if C // 8 <= 80 else 32)
    depth = C // lpr + 8                  # a lane's chain over its C / LPR values, then the xor tree
    gamma = Tin.view("gamma", F32, C).double()
    for r0 in range(0, M, rows):
        r1 = min(M, r0 + rows)
        X = Tin.view("x", BF16, M * C).view(M, C)[r0:r1].double()
        if spec["op"] == "pcm_layernorm_fwd":
            eps = f32(a["eps"])
            beta = Tin.view("beta", F32, C).double()
            m = X.mean(1, keepdim=True)
            v = (X - m).square().mean(1, keepdim=True)
            r = (v + eps).rsqrt()
            # mean: one chain of C values; var: (x - mean)^2 with the kernel's mean, so a mean error dm
            # adds dm^2 + 2 dm mean|x - m| on top of the chain's own error
            dm = depth * U * X.abs().mean(1, keepdim=True) + U * m.abs()
            dv = (depth + 2) * U * v + 2 * dm * (X - m).abs().mean(1, keepdim=True) + dm * dm
            dr = 0.5 * (dv + 2 * U * v) / (v + eps) + 6 * U
            if a["stats"]:
                st = Tout.view("stats", F32, 2 * M).view(M, 2)[r0:r1]
                yield Piece("ln stats", st[:, 0], m[:, 0], dm[:, 0])
                yield Piece("ln stats", st[:, 1], r[:, 0], (dr * r)[:, 0])
            ref = (X - m) * r * gamma + beta
            e = 4 * U * (((X - m) * r * gamma).abs() + beta.abs()) + gamma.abs() * r * (dm + (X - m).abs() * dr)
            yield Piece("ln fwd", Tout.view("out", BF16, M * C).view(M, C)[r0:r1], ref, bf16_bound(ref, e))
        else:
            st = Tin.view("stats", F32, 2 * M).view(M, 2)[r0:r1].double()
            m, r = st[:, :1], st[:, 1:]
            dy = Tin.view("dy", BF16, M * C).view(M, C)[r0:r1].double()
            g = dy * gamma
            xh = (X - m) * r
            s1, s2 = g.mean(1, keepdim=True), (g * xh).mean(1, keepdim=True)
            ad = Tin.view("add", BF16, M * C).view(M, C)[r0:r1].double() if a["add"] else 0.0
            ref = r * (g - s1 - xh * s2) + ad
            d1 = (depth + 1) * U * g.abs().mean(1, keepdim=True)
            d2 = (depth + 4) * U * (g * xh).abs().mean(1, keepdim=True)
            e = r * (d1 + xh.abs() * d2 + 4 * U * (g.abs() + s1.abs() + (xh * s2).abs())) + 2 * U * (ref - ad).abs()
            if a["add"]:
                e = e + U * (ref.abs() + ad.abs())
            yield Piece("ln bwd", Tout.view("dx", BF16, M * C).view(M, C)[r0:r1], ref, bf16_bound(ref, e))


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


def dgelu64(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def _geglu_ref(spec, Tin, Tout, rows=4096):
    a = spec["args"]
    M, Fh = a["M"], a["F"]
    for r0 in range(0, M, rows):
        r1 = min(M, r0 + rows)
        u = Tin.view("u", BF16, 2 * M * Fh).view(M, 2 * Fh)[r0:r1].double()
        x, g = u[:, :Fh], u[:, Fh:]
        erf = torch.erf(g / math.sqrt(2.0))
        # 0.5 g (1 + erff(g / sqrt2)) in fp32: erff to a few ulps, four roundings
        e_gelu = 0.5 * g.abs() * (U_FAST * erf.abs() + 4 * U * (1 + erf.abs()))
        if spec["op"] == "pcm_geglu_fwd":
            ref = x * gelu64(g)
            e = x.abs() * e_gelu + U * ref.abs()
            yield Piece("geglu fwd", Tout.view("out", BF16, M * Fh).view(M, Fh)[r0:r1], ref, bf16_bound(ref, e),
                        signed=x.sign(), e_fp32=e)
        else:
            d = Tin.view("dgg", BF16, M * Fh).view(M, Fh)[r0:r1].double()
            du = Tout.view("du", BF16, 2 * M * Fh).view(M, 2 * Fh)[r0:r1]
            ra = d * gelu64(g)
            ea = d.abs() * e_gelu + U * ra.abs()
            rg = d * x * dgelu64(g)
            # __expf(-g^2/2): (2 + 1.2 |g^2/2|) ulps
            phi = (g * torch.exp(-0.5 * g * g) / math.sqrt(2 * math.pi)).abs()
            e_d = 0.5 * (U_FAST * erf.abs() + 4 * U * (1 + erf.abs())) + phi * (2.0 ** -23 * (2 + 0.6 * g * g) + 4 * U)
            eg = (d * x).abs() * e_d + 2 * U * rg.abs()
            yield Piece("geglu bwd", du[:, :Fh], ra, bf16_bound(ra, ea), signed=d.sign(), e_fp32=ea)
            yield Piece("geglu bwd", du[:, Fh:], rg, bf16_bound(rg, eg), signed=(d * x).sign(), e_fp32=eg)


def upsample_bwd_exact(dout, B, H, W, C):
    """The kernel's fp32 sum of the four taps, (0,0) + (0,1) + (1,0) + (1,1), rounded once to bf16."""
    d = dout.view(B, H, 2, W, 2, C).float()
    s = d[:, :, 0, :, 0] + d[:, :, 0, :, 1]
    s = s + d[:, :, 1, :, 0]
    s = s + d[:, :, 1, :, 1]
    return s.to(BF16)


def _conv_ref(spec, Tin, Tout):
    import torch.nn.functional as F
    a = spec["args"]
    B, H, W, C = a["B"], a["H"], a["W"], a["C"]
    x = Tin.view("x", F32, B * H * W * 4).view(B, H, W, 4)
    xd = (x.to(BF16) if a["round_in"] else x).double().permute(0, 3, 1, 2)
    w = Tin.view("w", BF16, 36 * C).view(C, 3, 3, 4).double().permute(0, 3, 1, 2)
    if a["sgn"] < 0:
        w = w.flip(2, 3)
    bias = Tin.view("bias", F32, C).double() if a["bias"] else None
    out = Tout.view("out", BF16, B * H * W * C).view(B, H, W, C)
    for b in range(B):
        ref = F.conv2d(xd[b:b + 1], w, bias, padding=1)[0].permute(1, 2, 0)
        S = F.conv2d(xd[b:b + 1].abs(), w.abs(), None if bias is None else bias.abs(), padding=1)[0].permute(1, 2, 0)
        # 36 fp32 products added to the bias in one chain: 37 roundings of at most the sum of |terms|
        e = 38 * U * S
        yield Piece("conv_c4", out[b], ref, bf16_bound(ref, e))


def _timestep_ref(spec, Tin, Tout):
    a = spec["args"]
    B, C = a["B"], a["C"]
    half = C // 2
    t = Tin.view("t", torch.int64, B).double()
    k = torch.arange(half, device=t.device, dtype=F64)
    arg = t[:, None] * torch.exp(-math.log(10000.0) * k / half)[None]
    ref = torch.cat([arg.cos(), arg.sin()], 1)
    # expf of a rounded exponent, times t: the argument is within ~(4 + 9.3 k/half) u of itself; sincosf
    # adds a few ulps of its result
    e_arg = arg.abs() * U * (4 + 2 * 9.21 * k / half)
    e = torch.cat([e_arg, e_arg], 1) + U_FAST
    yield Piece("timestep", Tout.view("out", BF16, B * C).view(B, C), ref, bf16_bound(ref, e))


SLICE = 1 << 24            # elements per float64 reference slice of the flat optimiser buffers


def _slices(n):
    return ((i, min(n, i + SLICE)) for i in range(0, n, SLICE))


def sumsq64(x):
    """Sum of squares of a flat fp32 tensor in float64, one slice at a time."""
    return sum(float(x[i:j].double().square().sum()) for i, j in _slices(x.numel()))


def _adamw_ref(spec, Tin, Tout):
    """torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW restated in float64 from the fp32 state, one
    slice of the flat buffers at a time."""
    a = spec["args"]
    n = a["n"]
    b1, b2, eps, wd, mx, iw = (f32(a[k]) for k in ("beta1", "beta2", "eps", "wd", "max_norm", "inv_world"))
    st = Tin.view("state", F32, 2).double()
    lr, step = float(st[0]), float(st[1]) + 1.0
    norm = math.sqrt(float(Tin.view("sumsq", F64, 1)[0])) * iw
    coef = (min(mx / (norm + 1e-6), 1.0) if mx > 0 else 1.0) * iw
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    # fp32: coef within 6 u (sqrt of the double sum, divide, two products); powf to 4 ulps, which
    # 1 - beta^step magnifies by beta^step / (1 - beta^step); the update chain adds ~8 roundings
    dc = 6 * U
    r1 = 4 * U * b1 ** step / bc1 + 2 * U
    r2 = 4 * U * b2 ** step / bc2 + 2 * U
    ins = {k: Tin.view(k, F32, n) for k in ("p", "g", "m", "v")}
    outs = {k: Tout.view(k, F32, n) for k in ("p", "g", "m", "v")}
    for i, j in _slices(n):
        p, g, m, v = (ins[k][i:j].double() for k in ("p", "g", "m", "v"))
        gi = g * coef
        m1 = b1 * m + (1 - b1) * gi
        v1 = b2 * v + (1 - b2) * gi * gi
        den = v1.sqrt() / math.sqrt(bc2) + eps
        upd = lr / bc1 * m1 / den
        p1 = p * (1 - lr * wd) - upd
        em = 3 * U * (b1 * m.abs() + (1 - b1) * gi.abs()) + (1 - b1) * gi.abs() * dc
        ev = 3 * U * (b2 * v + (1 - b2) * gi * gi) + 2 * (1 - b2) * gi * gi * dc
        rden = (v1.sqrt() / math.sqrt(bc2) * (0.5 * ev / v1.clamp_min(1e-300) + 0.5 * r2 + 4 * U) + U * eps) / den
        rupd = r1 + em / m1.abs().clamp_min(1e-300) + rden + 4 * U
        ep = 3 * U * (p.abs() + p1.abs()) + upd.abs() * rupd
        yield Piece("adamw p", outs["p"][i:j], p1, ep)
        yield Piece("adamw m", outs["m"][i:j], m1, em + U * m1.abs())
        yield Piece("adamw v", outs["v"][i:j], v1, ev + U * v1)
        gref = torch.zeros(j - i, dtype=F32, device=g.device) if a["zero_grad"] else ins["g"][i:j]
        yield Piece("adamw g", outs["g"][i:j], gref)
    yield Piece("adamw state", Tout.view("state", F32, 2), torch.tensor([lr, step], dtype=F32, device=st.device))


def _refresh_ref(spec, Tin, Tout):
    a = spec["args"]
    scale = f32(a["scale"])
    master, opnd = Tin.view("master", F32), Tout.view("opnd", BF16)
    for e in _refresh_rows(spec["table"]):
        r, k, n, cin, taps = e["r"], e["taps"] * e["cin"], e["n"], e["cin"], e["taps"]
        A = master[e["a_off"]:e["a_off"] + r * k].view(r, k)
        sB = master[e["b_off"]:e["b_off"] + n * r].view(n, r) * scale        # fp32 product, as the kernel
        yield Piece("lora_refresh", opnd[e["a_fwd"]:e["a_fwd"] + r * k], A.to(BF16).reshape(-1))
        yield Piece("lora_refresh", opnd[e["a_t"]:e["a_t"] + r * k],
                    A.to(BF16).view(r, taps, cin).permute(2, 1, 0).reshape(-1))
        yield Piece("lora_refresh", opnd[e["sb_fwd"]:e["sb_fwd"] + n * r], sB.to(BF16).reshape(-1))
        yield Piece("lora_refresh", opnd[e["sb_t"]:e["sb_t"] + n * r], sB.to(BF16).t().reshape(-1))


def softmax_depth(cols):
    """Summation depth of one row sum of csrc/vae.cu softmax_rows_kernel: a float4's four exponentials are
    added pairwise (2), each thread chains its ceil(cols / 1024) float4s (256 threads of cols / 4 float4s),
    then the 5-level xor tree of a warp and the 8 warp partials added one after another (7)."""
    return -(-cols // 1024) + 2 + 5 + 7


def _softmax_ref(spec, Tin, Tout):
    """p = exp(s - max) / sum exp(s - max), bf16, against float64.

    The max is exact.  d = s - max is one fp32 subtraction (error u |d|, which exp turns into a relative
    u |d|); expf is within 2 ulps (2^-22 relative), plus 2^-149 where it underflows: e_j = exp(d_j) within
    r_j = (|d_j| + 4) u.  The sum of these positive terms passes through `softmax_depth` roundings, so the
    kernel's sum is within R = sum_j e_j r_j / sum + (depth + 1) u of the exact one (relative), the IEEE
    reciprocal and the product add u each: p_j in fp32 is within (r_j + R + 2 u)(1 + 2^-20) p_j + 2^-149
    of the exact value (the 2^-20 covers the products of first-order terms), then one bf16 rounding."""
    a = spec["args"]
    rows, cols = a["rows"], a["cols"]
    depth = softmax_depth(cols)
    s = softmax_scores(Tin)
    p = Tout.view("p", BF16).as_strided((rows, cols), (a["ldp"], 1))
    step = max(1, (1 << 22) // cols)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        x = s[r0:r1].double()
        d = x - x.max(1, keepdim=True).values
        e = d.exp()
        tot = e.sum(1, keepdim=True)
        r = (d.abs() + 4) * U
        R = (e * r).sum(1, keepdim=True) / tot + (depth + 1) * U
        ref = e / tot
        yield Piece("softmax", p[r0:r1], ref, bf16_bound(ref, (r + R + 2 * U) * (1 + 2.0 ** -20) * ref + 2.0 ** -149))


def _latent_ref(spec, Tin, Tout):
    """quant_conv and the latent distribution against float64.

    moments = bf16(sum_k bf16(h_k) w_k + bias): the first fma of the chain is exact (a product of two bf16
    values), the other 7 and the bias add round once each, so the fp32 value is within 8 u S of the exact
    sum, S = sum |h_k w_k| + |bias|; then one bf16 rounding.  logvar is that, clamped to [-30, 20]: both
    ends are bf16 values, so a moment past a clamp by more than its bound gives the clamp exactly.
    std = expf(logvar / 2) on the kernel's own logvar (checked first): the halving is exact, expf within
    2 ulps.  sample = (mean + std * noise) * scale, three fp32 roundings on the kernel's own mean and std:
    bit for bit the torch fp32 expression."""
    a = spec["args"]
    n = a["B"] * a["HW"]
    B, HW = a["B"], a["HW"]
    x = Tin.view("h", F32, 8 * n).view(n, 8).to(BF16).double()
    w = Tin.view("w", BF16, 64).view(8, 8).double()
    bias = Tin.view("bias", F32, 8).double()
    mo = x @ w.t() + bias
    e = 8 * U * (x.abs() @ w.abs().t() + bias.abs())

    def nchw(t):
        return t.view(B, HW, 4).permute(0, 2, 1)

    def out(name):
        return Tout.view(name, F32, 4 * n).view(B, 4, HW)
    yield Piece("latent_dist mean", out("mean"), nchw(mo[:, :4]), nchw(bf16_bound(mo[:, :4], e[:, :4])))
    lv = mo[:, 4:]
    bnd = bf16_bound(lv, e[:, 4:])
    clamped = lv.clamp(-30.0, 20.0)
    bnd = torch.where((clamped - lv).abs() > bnd, torch.zeros_like(bnd), bnd)
    yield Piece("latent_dist logvar", out("logvar"), nchw(clamped), nchw(bnd))
    sd = (out("logvar").double() / 2).exp()
    yield Piece("latent_dist std", out("std"), sd, 2.0 ** -22 * sd + 2.0 ** -149)
    if a["noise"]:
        noise = Tin.view("noise", F32, 4 * n).view(B, 4, HW)
        smp = (out("mean") + out("std") * noise) * torch.tensor(f32(a["scale"]), dtype=F32, device=noise.device)
        yield Piece("latent_dist sample", out("sample"), smp)


def _dec_in_ref(spec, Tin, Tout):
    """post_quant_conv on bf16(z / div) against float64: the input is the IEEE fp32 quotient rounded to
    bf16 (computed so here); the 4-term fma chain (the first product exact) and the bias add round 4 times,
    each within u S, S = sum |x_k w_k| + |bias|; then one bf16 rounding.  Channels 4..7 are zero, bit for bit."""
    a = spec["args"]
    M = a["M"]
    z = Tin.view("z", F32, 4 * M).view(M, 4)
    x = (z / torch.tensor(f32(a["div"]), dtype=F32, device=z.device)).to(BF16).double()
    w = Tin.view("w", BF16, 16).view(4, 4).double()
    bias = Tin.view("bias", F32, 4).double()
    ref = x @ w.t() + bias
    out = Tout.view("out", BF16, 8 * M).view(M, 8)
    yield Piece("vae_dec_in", out[:, :4], ref, bf16_bound(ref, 4 * U * (x.abs() @ w.abs().t() + bias.abs())))
    yield Piece("vae_dec_in zeros", out[:, 4:], torch.zeros(M, 4, dtype=BF16, device=z.device))


def _image_exit_ref(spec, Tin, Tout):
    """v = (x / 2 + 0.5).clamp(0, 1) and round(v * 255) in torch fp32 (x / 2 is exact, each other operation
    one IEEE rounding; round half to even): bit for bit, fp32 NCHW and uint8 NHWC."""
    a = spec["args"]
    B, HW, C = a["B"], a["HW"], a["C"]
    n = B * HW * C
    x = Tin.view("x", F32, n)
    for b in range(B):
        v = (x[b * HW * C:(b + 1) * HW * C] / 2 + 0.5).clamp(0.0, 1.0)
        if a["out"]:
            yield Piece("image_exit f32", Tout.view("out", F32, n).view(B, C, HW)[b], v.view(HW, C).t())
        if a["u8"]:
            yield Piece("image_exit u8", Tout.view("u8", torch.uint8, n).view(B, HW * C)[b], (v * 255).round().to(torch.uint8))


def reference(spec, Tin, Tout):
    """The Pieces of one launch: every output window of `Tout` against float64 (or exact) results computed
    from the inputs in `Tin` (a snapshot taken before the launch: AdamW and EMA update in place)."""
    op, a = spec["op"], spec["args"]
    if op in GN_OPS:
        yield from _gn_ref(spec, Tin, Tout)
    elif op.startswith("pcm_layernorm"):
        yield from _ln_ref(spec, Tin, Tout)
    elif op.startswith("pcm_geglu"):
        yield from _geglu_ref(spec, Tin, Tout)
    elif op == "pcm_upsample2x_fwd":
        B, H, W, C = a["B"], a["H"], a["W"], a["C"]
        x = Tin.view("x", BF16, B * H * W * C).view(B, H, W, C)
        ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1)
        yield Piece("upsample fwd", Tout.view("out", BF16, 4 * B * H * W * C), ref)
    elif op == "pcm_upsample2x_bwd":
        B, H, W, C = a["B"], a["H"], a["W"], a["C"]
        ref = upsample_bwd_exact(Tin.view("dout", BF16, 4 * B * H * W * C), B, H, W, C).reshape(-1)
        yield Piece("upsample bwd", Tout.view("din", BF16, B * H * W * C), ref)
    elif op == "pcm_conv3x3_c4":
        yield from _conv_ref(spec, Tin, Tout)
    elif op == "pcm_timestep_embed":
        yield from _timestep_ref(spec, Tin, Tout)
    elif op == "pcm_add_bf16":
        n = a["n"]
        x, y, out = Tin.view("a", BF16, n), Tin.view("b", BF16, n), Tout.view("out", BF16, n)
        for i, j in _slices(n):
            yield Piece("add_bf16", out[i:j], (x[i:j].float() + y[i:j].float()).to(BF16))
    elif op == "pcm_cast_f32_bf16":
        yield Piece("cast", Tout.view("out", BF16, a["n"]), Tin.view("x", F32, a["n"]).to(BF16))
    elif op == "pcm_grad_sumsq":
        s = torch.tensor([sumsq64(Tin.view("g", F32, a["n"]))], dtype=F64, device=Tin.device)
        # each float4 is squared and summed in fp32 (4 roundings of at most the quad's sum, i.e. 5 u of
        # it with the product roundings); the double accumulation adds < n 2^-53 of the total
        out = Tout.view("out", F64, 2)
        yield Piece("sumsq", out[:1], s, (5 * U + a["n"] * 2.0 ** -53) * s + 1e-300)
        yield Piece("sumsq counter", out[1:2].view(torch.int64), torch.zeros(1, dtype=torch.int64, device=s.device))
    elif op == "pcm_adamw_clip":
        yield from _adamw_ref(spec, Tin, Tout)
    elif op == "pcm_ema_update":
        n, rate = a["n"], f32(a["rate"])
        targ, src, out = Tin.view("targ", F32, n), Tin.view("src", F32, n), Tout.view("targ", F32, n)
        for i, j in _slices(n):
            t, s = targ[i:j].double(), src[i:j].double()
            ref = t * rate + s * f32(1 - rate)
            # 1 - rate is exact for rate in [1/2, 1]; two products and a sum
            yield Piece("ema", out[i:j], ref, 3 * U * ((t * rate).abs() + (s * (1 - rate)).abs())
                        + U * ref.abs() + (0 if rate >= 0.5 else U * s.abs()))
    elif op == "pcm_lora_refresh":
        yield from _refresh_ref(spec, Tin, Tout)
    elif op == "pcm_softmax_rows":
        yield from _softmax_ref(spec, Tin, Tout)
    elif op == "pcm_transpose_bf16":
        x, out = transpose_views(Tin)[0], transpose_views(Tout)[1]
        for b in range(a["batch"]):
            yield Piece("transpose", out[b], x[b].t())
    elif op == "pcm_latent_dist":
        yield from _latent_ref(spec, Tin, Tout)
    elif op == "pcm_vae_dec_in":
        yield from _dec_in_ref(spec, Tin, Tout)
    elif op == "pcm_image_exit":
        yield from _image_exit_ref(spec, Tin, Tout)
    else:
        raise KeyError(op)


SIGNED_K = 6.0


def check_piece(p):
    """Assert one Piece; returns its largest err / bound (0 for a bitwise piece).

    Bitwise pieces compare the bit patterns (NaN payloads included).  Bounded pieces must be finite and
    within the bound elementwise.  A piece with `signed` weights w also passes the signed error test, which
    resolves a formula error far below one ulp per element (tanh-GELU against erf-GELU): the output is
    compared with the correctly rounded reference RNE(ref).  The kernel's fp32 value is within e_fp32 of ref,
    so it rounds differently only near a rounding boundary, by one ulp, up or down as its fp32 error falls;
    an unbiased error makes those differences d a zero-mean sum, a bias b per element adds at most b each.
    So |sum w d| <= SIGNED_K sqrt(sum d^2) + sum e_fp32, whereas a formula off by a fraction of an ulp
    moves many roundings the same way.  (RNE(ref) itself is not compared with ref: where the density of
    the values falls off within an ulp, correct roundings are biased by a fraction of an ulp too.)"""
    got = p.got
    if p.bnd is None:
        ref = p.ref.to(got.dtype).reshape(got.shape)
        if got.dtype.is_floating_point:
            bits = {2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
            gb, rb = got.view(bits), ref.view(bits)
        else:
            gb, rb = got, ref
        bad = gb != rb
        if bad.any():
            i = int(bad.reshape(-1).nonzero()[0])
            raise AssertionError(f"{p.fam}: {int(bad.sum())} of {bad.numel()} elements differ bitwise, first at "
                                 f"{i}: got {got.reshape(-1)[i].item()!r} want {ref.reshape(-1)[i].item()!r}")
        return 0.0
    out = got.double().reshape(p.ref.shape)
    fin = torch.isfinite(out)
    if not fin.all():
        i = int((~fin).reshape(-1).nonzero()[0])
        raise AssertionError(f"{p.fam}: {int((~fin).sum())} non-finite elements of {out.numel()}, first at {i}")
    err = (out - p.ref).abs()
    ratio = err / (p.bnd + 1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError(f"{p.fam}: {int((ratio > 1).sum())} of {ratio.numel()} elements outside the bound, worst at "
                             f"{i}: got {float(out.reshape(-1)[i])!r} ref {float(p.ref.reshape(-1)[i])!r} bound "
                             f"{float(p.bnd.reshape(-1)[i]):.3e} (x{worst:.2f})")
    if p.signed is not None:
        d = out - p.ref.to(got.dtype).double()
        s = float((d * p.signed).sum())
        lim = SIGNED_K * math.sqrt(float(d.square().sum())) + float(p.e_fp32.sum())
        if abs(s) > lim:
            raise AssertionError(f"{p.fam}: signed error sum {s:.3e} exceeds {lim:.3e} "
                                 f"(a bias of {s / out.numel():.2e} per element)")
    return worst


def check(spec, Tin, Tout):
    """Check every output window of a launch; returns {family: largest err / bound}."""
    worst = {}
    for p in reference(spec, Tin, Tout):
        w = check_piece(p)
        worst[p.fam] = max(worst.get(p.fam, 0.0), w)
    return worst


# ---------------------------------------------------------------------------------------------
# launching (GPU tests) and guards
# ---------------------------------------------------------------------------------------------
def call_args(spec, T, **over):
    """The C ABI arguments of a spec on materialised buffers (stream excluded), exactly as recorded
    except the GroupNorm workspace (T.ws) and any `over`ride."""
    out = []
    for k in ARGS[spec["op"]]:
        if k in over:
            out.append(over[k])
        elif k == "ws":
            out.append(T.ws.data_ptr() if T.ws is not None and T.ws.numel() else 0)
        elif k == "ws_bytes":
            out.append(T.ws.numel() if T.ws is not None else 0)
        elif isinstance(spec["args"][k], list) or spec["args"][k] is None:
            out.append(T.addr(k))
        else:
            out.append(spec["args"][k])
    return out


def launch(spec, T, **over):
    """Launch through the C ABI on torch's current stream; returns the return code (0: launched)."""
    from pcm_b200 import _lib
    fn = getattr(_lib.lib(), spec["op"])
    return fn(*call_args(spec, T, **over), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def out_windows(spec):
    """(label, first byte, bytes) of every window the launch may write.  A strided output (softmax rows
    ldp apart, transposed rows ldo / bso apart) is one window per row when its rows leave gutters."""
    op, a = spec["op"], spec["args"]
    ext = extents(op, a, spec.get("table"))
    wins = []
    for k in _OUTS[op]:
        if not isinstance(a.get(k), list):
            continue
        lab, off = a[k]
        if op == "pcm_softmax_rows" and a["ldp"] != a["cols"]:
            wins += [(lab, off + 2 * r * a["ldp"], 2 * a["cols"]) for r in range(a["rows"])]
        elif op == "pcm_transpose_bf16" and (a["ldo"] != a["rows"] or a["bso"] != a["cols"] * a["rows"]):
            wins += [(lab, off + 2 * (b * a["bso"] + c * a["ldo"]), 2 * a["rows"])
                     for b in range(a["batch"]) for c in range(a["cols"])]
        else:
            wins.append((lab, off, ext[k]))
    return wins


def guards(spec, T, before):
    """Outside the output windows every byte of every buffer is what it was before the launch (checked one
    buffer at a time: the optimiser's buffers are 0.8 GB each)."""
    wins = out_windows(spec)
    for lab, (b, b0) in enumerate(zip(T.bufs, before.bufs)):
        changed = b != b0
        for wl, off, n in wins:
            if wl == lab:
                assert off % 2 == 0
                changed[off // 2:(off + n + 1) // 2] = False
        if changed.any():
            at = changed.nonzero().flatten()
            raise AssertionError(f"{spec['op']} buffer {lab}: {len(at)} 2-byte words outside the output windows "
                                 f"changed, byte offsets {2 * int(at[0])}..{2 * int(at[-1])} (span {spec['spans'][lab]})")
