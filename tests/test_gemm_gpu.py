"""Parity of the wgmma implicit GEMM (pcm_gemm / pcm_wgrad) against plain PyTorch fp32 ops
(F.linear / F.conv2d on bf16-rounded inputs).  Tolerance: outputs are bf16 (rel 2^-9 rounding),
accumulation fp32 -> |err| <= 1e-2 * max|ref| elementwise and mean error <= 2e-3 * rms(ref)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _close(out, ref, tol=1e-2):
    out, ref = out.float(), ref.float()
    err = (out - ref).abs()
    scale = ref.abs().max().item() + 1e-6
    rms = ref.pow(2).mean().sqrt().item() + 1e-6
    assert err.max().item() <= tol * scale, (err.max().item(), scale)
    assert err.mean().item() <= 2e-3 * rms + 1e-6, (err.mean().item(), rms)


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(torch.bfloat16)


def _wmat_conv(w):
    """[O, I, kh, kw] -> [O, (kh, kw, I)] tap-major K layout used by the K program."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


@pytest.mark.parametrize("M,K,N", [(616, 768, 320), (4096, 320, 1280), (128, 64, 64), (8, 1280, 320)])
def test_linear(cuda, M, K, N):
    from pcm_b200 import ops
    x = _rand((M, K), cuda, 1)
    w = _rand((N, K), cuda, 2, K ** -0.5)
    bias = torch.randn(N, device=cuda)
    res = _rand((M, N), cuda, 3)
    out = torch.empty(M, N, device=cuda, dtype=torch.bfloat16)
    ops.gemm([ops.asrc_mat(x)], [ops.bsrc(w)], [(0, 0, 0, 0, K // 64, 0, 0)], lin=True, M=M, N=N,
             out=out, bias=bias, residual=res, alpha=0.5)
    ref = 0.5 * F.linear(x.float(), w.float()) + bias + res.float()
    _close(out, ref)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 32, 32, 128, 192), (3, 8, 8, 64, 96), (1, 4, 4, 64, 32),
                                            (2, 64, 64, 64, 320), (2, 16, 16, 192, 64)])
def test_conv3x3(cuda, B, H, W, Cin, Cout):
    from pcm_b200 import ops
    x = _rand((B, H, W, Cin), cuda, 1)
    w = _rand((Cout, Cin, 3, 3), cuda, 2, (9 * Cin) ** -0.5)
    bias = torch.randn(Cout, device=cuda)
    rowvec = _rand((B, Cout), cuda, 4)
    out = torch.empty(B, H, W, Cout, device=cuda, dtype=torch.bfloat16)
    prog = [(0, 0, dw, dh, Cin // 64, 0, t * Cin) for t, (dw, dh) in enumerate(ops.TAPS3)]
    wm = _wmat_conv(w)
    ops.gemm([ops.asrc_nhwc(x)], [ops.bsrc(wm)], prog, lin=False, M=B * H * W, N=Cout,
             geo=(W, H), out=out.view(-1, Cout), bias=bias, rowvec=rowvec)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    ref = ref + rowvec.float()[:, :, None, None]
    _close(out.permute(0, 3, 1, 2), ref)


def test_conv_concat_lora_fp32out(cuda):
    """Two K segments (skip-concat) + LoRA up-projection segment, fp32 output."""
    from pcm_b200 import ops
    B, H, W, C1, C2, Cout = 2, 16, 16, 128, 64, 160
    x1, x2 = _rand((B, H, W, C1), cuda, 1), _rand((B, H, W, C2), cuda, 2)
    w = _rand((Cout, C1 + C2, 3, 3), cuda, 3, (9 * (C1 + C2)) ** -0.5)
    t = _rand((B, H, W, 64), cuda, 4)
    sb = _rand((Cout, 64), cuda, 5, 0.05)
    w1, w2 = _wmat_conv(w[:, :C1]), _wmat_conv(w[:, C1:])
    wcat = torch.cat([w1, w2], 1).contiguous()
    prog = [(0, 0, dw, dh, C1 // 64, 0, i * C1) for i, (dw, dh) in enumerate(ops.TAPS3)]
    prog += [(1, 0, dw, dh, C2 // 64, 0, 9 * C1 + i * C2) for i, (dw, dh) in enumerate(ops.TAPS3)]
    prog += [(2, 1, 0, 0, 1, 0, 0)]
    out = torch.empty(B * H * W, Cout, device=cuda, dtype=torch.float32)
    ops.gemm([ops.asrc_nhwc(x1), ops.asrc_nhwc(x2), ops.asrc_nhwc(t)], [ops.bsrc(wcat), ops.bsrc(sb)],
             prog, lin=False, M=B * H * W, N=Cout, geo=(W, H), out=out)
    xin = torch.cat([x1, x2], -1).float().permute(0, 3, 1, 2)
    ref = F.conv2d(xin, w.float(), padding=1) + (t.float().view(-1, 64) @ sb.float().t()).view(B, H, W, Cout).permute(0, 3, 1, 2)
    _close(out.view(B, H, W, Cout).permute(0, 3, 1, 2), ref, tol=2e-3)


def test_conv_stride2_parity_planes(cuda):
    """3x3 stride-2 pad-1 convolution expressed with four parity-plane A sources."""
    from pcm_b200 import ops
    B, H, W, Cin, Cout = 2, 32, 32, 64, 128
    x = _rand((B, H, W, Cin), cuda, 1)
    w = _rand((Cout, Cin, 3, 3), cuda, 2, (9 * Cin) ** -0.5)
    planes = [x[:, p::2, q::2, :] for p in range(2) for q in range(2)]  # index p*2+q
    prog = []
    for kh in range(3):
        for kw in range(3):
            p, dh = ((1, -1), (0, 0), (1, 0))[kh]
            q, dw = ((1, -1), (0, 0), (1, 0))[kw]
            prog.append((p * 2 + q, 0, dw, dh, Cin // 64, 0, (kh * 3 + kw) * Cin))
    out = torch.empty(B, H // 2, W // 2, Cout, device=cuda, dtype=torch.bfloat16)
    wm = _wmat_conv(w)
    ops.gemm([ops.asrc_nhwc(pl) for pl in planes], [ops.bsrc(wm)], prog, lin=False,
             M=B * H * W // 4, N=Cout, geo=(W // 2, H // 2), out=out.view(-1, Cout))
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), stride=2, padding=1)
    _close(out.permute(0, 3, 1, 2), ref)


def test_wgrad_linear(cuda):
    from pcm_b200 import ops
    M, Cp = 1000, 320
    p = _rand((M, Cp), cuda, 1)
    q = _rand((M, 64), cuda, 2)
    out = torch.zeros(Cp, 64, device=cuda)
    ops.wgrad(ops.asrc_mat(p), ops.asrc_mat(q), out, lin=True, M=M, os_row=64, os_col=1, alpha=0.125)
    ref = 0.125 * p.float().t() @ q.float()
    _close(out, ref, tol=2e-3)
    # transposed destination: out2[r, ch]
    out2 = torch.zeros(64, Cp, device=cuda)
    ops.wgrad(ops.asrc_mat(p), ops.asrc_mat(q), out2, lin=True, M=M, os_row=1, os_col=Cp)
    _close(out2, (p.float().t() @ q.float()).t(), tol=2e-3)


def test_wgrad_conv_taps(cuda):
    """dA[r, tap, c] = sum_m dt[m, r] * x[m + tap, c] for a 3x3 LoRA-A convolution."""
    from pcm_b200 import ops
    B, H, W, Cin = 2, 16, 16, 128
    x = _rand((B, H, W, Cin), cuda, 1)
    dt = _rand((B, H, W, 64), cuda, 2)
    out = torch.zeros(64, 9, Cin, device=cuda)
    ops.wgrad(ops.asrc_nhwc(x), ops.asrc_nhwc(dt), out, lin=False, M=B * H * W, geo=(W, H),
              taps=ops.TAPS3, tap_off=[t * Cin for t in range(9)], os_row=1, os_col=9 * Cin)
    xf = x.float().permute(0, 3, 1, 2).requires_grad_(False)
    a = torch.zeros(64, Cin, 3, 3, device=cuda, requires_grad=True)
    y = F.conv2d(xf, a, padding=1)
    y.backward(dt.float().permute(0, 3, 1, 2))
    ref = a.grad.permute(0, 2, 3, 1).reshape(64, 9, Cin)
    _close(out, ref, tol=2e-3)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(8, 8, 8, 1280, 1280), (8, 8, 8, 1280, 64), (2, 16, 16, 640, 64)])
def test_conv3x3_splitk(cuda, B, H, W, Cin, Cout):
    """Small-M long-K convolutions run split-K (per-split fp32 workspace slices + ordered finalize)."""
    from pcm_b200 import ops
    x = _rand((B, H, W, Cin), cuda, 1)
    w = _rand((Cout, Cin, 3, 3), cuda, 2, (9 * Cin) ** -0.5)
    bias = torch.randn(Cout, device=cuda)
    res = _rand((B, H, W, Cout), cuda, 5)
    rowvec = _rand((B, Cout), cuda, 4)
    out = torch.empty(B, H, W, Cout, device=cuda, dtype=torch.bfloat16)
    prog = [(0, 0, dw, dh, Cin // 64, 0, t * Cin) for t, (dw, dh) in enumerate(ops.TAPS3)]
    M = B * H * W
    bn, ks = ops.pick_tiling(M, Cout, len(prog) * (Cin // 64))
    assert ks > 1
    # (the weight copy must outlive the launch: ops.bsrc() only takes its device pointer, and a
    # temporary's memory could be handed to the split-K workspace allocated inside ops.gemm)
    wm = _wmat_conv(w)
    ops.gemm([ops.asrc_nhwc(x)], [ops.bsrc(wm)], prog, lin=False, M=M, N=Cout,
             geo=(W, H), out=out.view(-1, Cout), bias=bias, rowvec=rowvec, residual=res.view(-1, Cout), act=1)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    ref = F.silu(ref + rowvec.float()[:, :, None, None] + res.float().permute(0, 3, 1, 2))
    _close(out.permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize("M,Ml,K,C,g", [(1848, 616, 768, 320, 2), (4096, 2048, 320, 320, 3), (300, 300, 128, 64, 3)])
def test_grouped_linear_n_ranges(cuda, M, Ml, K, C, g):
    """g Linear layers sharing their input as one GEMM (N = g*C): per-layer LoRA K blocks restricted
    to their own output columns by N-ranged K entries; only the first Ml rows carry the adapter
    (T has Ml rows, the rest is TMA zero fill); 4 B sources in the dgrad-style second launch."""
    from pcm_b200 import ops
    x = _rand((M, K), cuda, 1)
    w = _rand((g * C, K), cuda, 2, K ** -0.5)
    T = _rand((Ml, g * 64), cuda, 3)
    sb = _rand((g * C, 64), cuda, 4, 0.1)
    bn = 160 if C % 160 == 0 else 64
    prog = [(0, 0, 0, 0, K // 64, 0, 0)] + [(1, 1, 0, 0, 1, i * 64, 0, i * C, (i + 1) * C) for i in range(g)]
    out = torch.empty(M, g * C, device=cuda, dtype=torch.bfloat16)
    ops.gemm([ops.asrc_mat(x), ops.asrc_mat(T)], [ops.bsrc(w), ops.bsrc(sb)], prog, lin=True, M=M, N=g * C,
             out=out, block_n=bn)
    ref = F.linear(x.float(), w.float())
    for i in range(g):
        ref[:Ml, i * C:(i + 1) * C] += T[:, i * 64:(i + 1) * 64].float() @ sb[i * C:(i + 1) * C].float().t()
    _close(out, ref)
    # N-ranged A column blocks (the dT = dy_i @ (sB_i) launch) reading column views of `out`
    sbt = _rand((g * 64, C), cuda, 5, C ** -0.5)
    dT = torch.empty(M, g * 64, device=cuda, dtype=torch.bfloat16)
    prog = [(0, 0, 0, 0, C // 64, i * C, 0, i * 64, (i + 1) * 64) for i in range(g)]
    ops.gemm([ops.asrc_mat(out)], [ops.bsrc(sbt)], prog, lin=True, M=M, N=g * 64, out=dT, block_n=64)
    ref2 = torch.cat([out[:, i * C:(i + 1) * C].float() @ sbt[i * 64:(i + 1) * 64].float().t() for i in range(g)], 1)
    _close(dT, ref2)
    # 1 + g B sources
    wt = _rand((K, g * C), cuda, 6, (g * C) ** -0.5)
    ats = [_rand((K, 64), cuda, 7 + i, 0.1) for i in range(g)]
    prog = [(0, 0, 0, 0, g * C // 64, 0, 0)] + [(1, 1 + i, 0, 0, 1, i * 64, 0) for i in range(g)]
    dx = torch.empty(M, K, device=cuda, dtype=torch.bfloat16)
    ops.gemm([ops.asrc_mat(out), ops.asrc_mat(dT)], [ops.bsrc(wt)] + [ops.bsrc(a) for a in ats], prog, lin=True,
             M=M, N=K, out=dx)
    ref3 = out.float() @ wt.float().t()
    for i in range(g):
        ref3 += dT[:, i * 64:(i + 1) * 64].float() @ ats[i].float().t()
    _close(dx, ref3)


@pytest.mark.parametrize("kind,shape", [("lin", (616, 768, 320)), ("conv", (2, 16, 16, 192, 96)), ("conv", (8, 8, 8, 1280, 256))])
def test_kblocked_weights_bit_identical(cuda, kind, shape):
    """K-blocked weight storage ([K/64][N][64], pcm_bsrc.kblocked) is a pure re-layout: same tiles, same
    MMA order -> bit-identical output to the row-major source, also mixed with a row-major second source
    (the LoRA s*B operand) in one K program, and through split-K."""
    from pcm_b200 import ops
    if kind == "lin":
        M, K, N = shape
        x = _rand((M, K), cuda, 1)
        w = _rand((N, K), cuda, 2, K ** -0.5)
        t = _rand((M, 64), cuda, 3)
        sb = _rand((N, 64), cuda, 4, 0.1)
        srcs = [ops.asrc_mat(x), ops.asrc_mat(t)]
        prog = [(0, 0, 0, 0, K // 64, 0, 0), (1, 1, 0, 0, 1, 0, 0)]
        kw = dict(lin=True, M=M, N=N)
        ref = F.linear(x.float(), w.float()) + F.linear(t.float(), sb.float())
    else:
        B, H, W, Cin, N = shape
        M = B * H * W
        x = _rand((B, H, W, Cin), cuda, 1)
        w4 = _rand((N, Cin, 3, 3), cuda, 2, (9 * Cin) ** -0.5)
        w = _wmat_conv(w4)
        t = _rand((B, H, W, 64), cuda, 3)
        sb = _rand((N, 64), cuda, 4, 0.1)
        srcs = [ops.asrc_nhwc(x), ops.asrc_nhwc(t)]
        prog = [(0, 0, dw, dh, Cin // 64, 0, tt * Cin) for tt, (dw, dh) in enumerate(ops.TAPS3)] + [(1, 1, 0, 0, 1, 0, 0)]
        kw = dict(lin=False, M=M, N=N, geo=(W, H))
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w4.float(), None, padding=1).permute(0, 2, 3, 1).reshape(M, N)
        ref = ref + F.linear(t.float().reshape(M, 64), sb.float())
    wb = ops.kblock(w)
    assert wb.shape == (w.shape[1] // 64, w.shape[0], 64)
    o1 = torch.empty(M, N, device=cuda, dtype=torch.bfloat16)
    o2 = torch.empty_like(o1)
    ops.gemm(srcs, [ops.bsrc(w), ops.bsrc(sb)], prog, out=o1, **kw)
    ops.gemm(srcs, [ops.bsrc(wb), ops.bsrc(sb)], prog, out=o2, **kw)
    torch.cuda.synchronize()
    _close(o1, ref)
    assert torch.equal(o1, o2)
