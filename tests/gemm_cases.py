"""Builders of synthetic pcm_gemm / pcm_wgrad specs and the GPU run-and-check step, shared by
test_gemm_specs_cpu.py, test_gemm_prod_gpu.py and test_gemm_edges_gpu.py.  A spec is built by recording the
ops.gemm / ops.wgrad call on empty CPU tensors, so its descriptor is the one the Python wrappers produce."""
import torch

import gemm_spec as G

BF16, F32 = torch.bfloat16, torch.float32
# stride-2 3x3 pad-1: kernel index -> (input parity, shift in that parity plane)
S2 = ((1, -1), (0, 0), (1, 0))


def empty(shape, dtype=BF16):
    return torch.empty(shape, dtype=dtype)


def build(fn):
    """The spec of the last launch `fn(ops)` issues on CPU tensors (with its producer when it has dep_a_src)."""
    from pcm_b200 import ops
    with G.recording() as rec:
        fn(ops)
        recs = [r for r in rec.trace if r["op"] in ("gemm", "wgrad")]
    last = recs[-1]
    dep = last["op"] == "gemm" and last["desc"]["dep_a_src1"]
    return G.spec_of(last, recs[-2] if dep else None)


def conv3x3_spec(B=2, H=8, W=8, Cin=64, Cout=96, rowvec=False, residual=False, **kw):
    def fn(ops):
        M = B * H * W
        prog = [(0, 0, dw, dh, Cin // 64, 0, t * Cin) for t, (dw, dh) in enumerate(ops.TAPS3)]
        ops.gemm([ops.asrc_nhwc(empty((B, H, W, Cin)))], [ops.bsrc(empty((Cout, 9 * Cin)))], prog, lin=False, M=M,
                 N=Cout, geo=(W, H), out=empty((M, Cout)), bias=empty((Cout,), F32),
                 rowvec=empty((B, Cout + 8))[:, :Cout] if rowvec else None,
                 residual=empty((M, Cout)) if residual else None, **kw)
    return build(fn)


def stride2_spec(B=2, H=8, W=8, Cin=64, Cout=64):
    """3x3 stride-2 pad-1 convolution reading the four parity planes of its input."""
    def fn(ops):
        x = empty((B, H, W, Cin))
        planes = [x[:, p::2, q::2, :] for p in range(2) for q in range(2)]
        prog = [(S2[kh][0] * 2 + S2[kw][0], 0, S2[kw][1], S2[kh][1], Cin // 64, 0, (kh * 3 + kw) * Cin)
                for kh in range(3) for kw in range(3)]
        ops.gemm([ops.asrc_nhwc(p) for p in planes], [ops.bsrc(empty((Cout, 9 * Cin)))], prog, lin=False,
                 M=B * H * W // 4, N=Cout, geo=(W // 2, H // 2), out=empty((B * H * W // 4, Cout)))
    return build(fn)


def dgrad2_spec(p, q, B=2, H=8, W=8, Cin=64, Cout=64, rank=0):
    """Input gradient of that convolution for parity plane (p, q) of dx [B, H, W, Cin]: flipped taps of
    dy [B, H/2, W/2, Cout] against W^T [Cin, (tap, Cout)], stored through out_strides / epi into the plane
    (the other three planes and the channel gutter are not this launch's).  rank: a LoRA block on top."""
    def fn(ops):
        Ho, Wo = H // 2, W // 2
        taps = [(kh * 3 + kw, -sw, -sh) for kh, (ph, sh) in enumerate(S2) if ph == p
                for kw, (pw, sw) in enumerate(S2) if pw == q]
        a, b = [ops.asrc_nhwc(empty((B, Ho, Wo, Cout)))], [ops.bsrc(empty((Cin, 9 * Cout)))]
        prog = [(0, 0, dw, dh, Cout // 64, 0, t * Cout) for t, dw, dh in taps]
        if rank:
            a.append(ops.asrc_nhwc(empty((B, Ho, Wo, rank))))
            b.append(ops.bsrc(empty((Cin, 9 * rank))))
            prog += [(1, 1, dw, dh, -(-rank // 64), 0, t * rank) for t, dw, dh in taps]
        plane = empty((B, H, W, Cin + 8))[:, p::2, q::2, :Cin]
        ops.gemm(a, b, prog, lin=False, M=B * Ho * Wo, N=Cin, geo=(Wo, Ho), out=plane,
                 out_strides=(plane.stride(2), plane.stride(1), plane.stride(0)), epi=(Wo, Wo * Ho))
    return build(fn)


def concat_lora_spec(B=2, H=8, W=8, C1=128, C2=64, Cout=96, r=24):
    def fn(ops):
        x1, x2, t = empty((B, H, W, C1)), empty((B, H, W, C2)), empty((B, H, W, r))
        w, sb, out = empty((Cout, 9 * (C1 + C2))), empty((Cout, r)), empty((B * H * W, Cout), F32)
        prog = [(0, 0, dw, dh, C1 // 64, 0, i * C1) for i, (dw, dh) in enumerate(ops.TAPS3)]
        prog += [(1, 0, dw, dh, C2 // 64, 0, 9 * C1 + i * C2) for i, (dw, dh) in enumerate(ops.TAPS3)]
        prog += [(2, 1, 0, 0, 1, 0, 0)]
        ops.gemm([ops.asrc_nhwc(x1), ops.asrc_nhwc(x2), ops.asrc_nhwc(t)], [ops.bsrc(w), ops.bsrc(sb)], prog,
                 lin=False, M=B * H * W, N=Cout, geo=(W, H), out=out)
    return build(fn)


def grouped_spec(M=300, Ml=128, K=128, C=64, g=3):
    """g Linear layers sharing their input, each with its own N-ranged LoRA block on the first Ml rows."""
    def fn(ops):
        x, w, T, sb, out = empty((M, K)), empty((g * C, K)), empty((Ml, g * 64)), empty((g * C, 64)), empty((M, g * C))
        prog = [(0, 0, 0, 0, K // 64, 0, 0)] + [(1, 1, 0, 0, 1, i * 64, 0, i * C, (i + 1) * C) for i in range(g)]
        ops.gemm([ops.asrc_mat(x), ops.asrc_mat(T)], [ops.bsrc(w), ops.bsrc(sb)], prog, lin=True, M=M, N=g * C,
                 out=out, block_n=64, residual=empty((M, g * C)))
    return build(fn)


def linear_spec(M=200, K=256, N=96, *, block_n=None, rank=0, Ml=None, ksplit=None, bias=True, rowvec=False,
                residual=True, inplace=False, act=0, out="bf16", alpha=1.0, window=None, dep=False, ranged=None,
                gutter=0):
    """One Linear launch: x [M, K] (window = (width, c0): a column window of a wider matrix), an optional
    LoRA block of `rank` on the first Ml rows (dep: produced by the launch immediately before; ranged =
    (n_lo, n_hi): only feeding those columns), output rows `gutter` elements apart beyond N rounded to 8."""
    def fn(ops):
        ld = (N + 7) // 8 * 8 + gutter if gutter else N
        o = empty((M, ld), F32 if out != "bf16" else BF16)[:, :N]
        wide, c0 = window or (K, 0)
        x = empty((M, wide))[:, c0:c0 + K]
        a, b = [ops.asrc_mat(x)], [ops.bsrc(empty((N, K)))]
        prog = [(0, 0, 0, 0, K // 64, 0, 0)]
        kw = {}
        if rank:
            t = empty((Ml or M, rank))
            if dep:
                ops.gemm([ops.asrc_mat(x)], [ops.bsrc(empty((rank, K)))], [(0, 0, 0, 0, K // 64, 0, 0)], lin=True,
                         M=Ml or M, N=rank, out=t, block_n=32 if rank < 64 else 64)
                kw["dep_a_src"] = 1
            a.append(ops.asrc_mat(t))
            b.append(ops.bsrc(empty((N, rank))))
            e = (1, 1, 0, 0, -(-rank // 64), 0, 0)
            prog.append(e + tuple(ranged) if ranged else e)
        res = o if inplace else (empty((M, ld))[:, :N] if residual else None)
        ops.gemm(a, b, prog, lin=True, M=M, N=N, out=o, block_n=block_n, ksplit=ksplit,
                 bias=empty((N,), F32) if bias else None, rowvec=empty((1, N + 8))[:, :N] if rowvec else None,
                 residual=res, act=act, alpha=alpha, round_bf16=out == "round", **kw)
    return build(fn)


def wgrad_spec(lin, M=300, Cp=96, qC=64, q_c0=0, B=2, H=8, W=8, **kw):
    """Linear: out[ch, r] (ranks contiguous).  Conv: the 9 taps of a 3x3 LoRA-A gradient, out[r, tap, ch]."""
    def fn(ops):
        qw = min(64, qC - q_c0)
        if lin:
            ops.wgrad(ops.asrc_mat(empty((M, Cp))), ops.asrc_mat(empty((M, qC))), empty((Cp, qw), F32), lin=True, M=M,
                      q_c0=q_c0, os_row=qw, os_col=1, **kw)
        else:
            ops.wgrad(ops.asrc_nhwc(empty((B, H, W, Cp))), ops.asrc_nhwc(empty((B, H, W, qC))), empty((qw, 9, Cp), F32),
                      lin=False, M=B * H * W, geo=(W, H), taps=ops.TAPS3, tap_off=[t * Cp for t in range(9)], os_row=1,
                      os_col=9 * Cp, q_c0=q_c0, **kw)
    return build(fn)


# ---------------------------------------------------------------------------------------------
# one launch on the GPU
# ---------------------------------------------------------------------------------------------
MARGIN = {}     # launch family -> (largest err / bound, largest k16 step count) of this session


def restore(T, before):
    for b, b0 in zip(T.bufs, before):
        b.copy_(b0)


def result(spec, T):
    flat, idx = G.window(spec, T)
    return flat[idx]


def run_and_check(spec, T, before, **kw):
    """Launch, compare with the float64 reference of the operands as the launch read them, check the guards
    and, for split-K, that every workspace element the finalize kernel reads was written."""
    G.launch(spec, T, **kw)
    torch.cuda.synchronize()
    out = result(spec, T)
    after = G.snapshot(T)
    if "pre" in spec or spec["op"] == "wgrad" or spec["desc"]["residual"] == spec["desc"]["out"]:
        # the reference reads what the launch read: the intermediate its producer wrote, the old destination
        mid = None
        if "pre" in spec:
            flat, idx = G.window(dict(op="gemm", desc=spec["pre"]), T)
            mid = flat[idx].clone()
            assert torch.isfinite(mid.float()).all()
        restore(T, before)
        if mid is not None:
            flat[idx] = mid
    ref, S, base = (G.reference_wgrad if spec["op"] == "wgrad" else G.reference)(spec, T)
    restore(T, after)
    worst = G.check(out, ref, S, spec, base=base)
    G.guards(spec, T, before)
    if spec["op"] == "gemm" and T.ws is not None:
        ks = G.resolved_ksplit(spec["desc"])
        n = (ks if ks > 1 else 0) * spec["desc"]["M"] * spec["desc"]["N"]     # an unsplit launch leaves it alone
        assert torch.isfinite(T.ws[:n]).all(), "a split-K slice element the finalize kernel reads was never written"
        assert T.ws[n:].isnan().all()
    fam, steps = G.family(spec), sum(G.k_steps(spec))
    w0, s0 = MARGIN.get(fam, (0.0, 0))
    MARGIN[fam] = (max(w0, worst), max(s0, steps))
    return out


def run(spec, device, seed=0, **kw):
    T = G.materialise(spec, device, seed)
    return run_and_check(spec, T, G.snapshot(T), **kw)


def report(title):
    """The margins of this session so far, per launch family, with the longest sum: the accumulate term of
    the bound grows linearly with the k16 steps, so a family's test is the less sensitive the longer its K."""
    lines = [title] + [f"  largest err / bound {w:.3f}  (up to {s} k16 steps + partial sums)  {fam}"
                       for fam, (w, s) in sorted(MARGIN.items())]
    return "\n".join(lines)
