"""Parity of the HBM-bound kernels against plain PyTorch fp32 (autograd for the backward passes);
the flash attention kernels are tested in test_attn_gpu.py.  Inputs are bf16-rounded; outputs are bf16 -> tolerance
1e-2 of the tensor's max magnitude elementwise and 3e-3 * rms mean error."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _close(out, ref, tol=1e-2, mtol=3e-3):
    out, ref = out.float(), ref.float()
    assert torch.isfinite(out).all()
    err = (out - ref).abs()
    scale = ref.abs().max().item() + 1e-6
    rms = ref.pow(2).mean().sqrt().item() + 1e-6
    assert err.max().item() <= tol * scale, (err.max().item(), scale)
    assert err.mean().item() <= mtol * rms + 1e-6, (err.mean().item(), rms)


def _rand(shape, dev, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + shift).to(dev).to(BF)


@pytest.mark.parametrize("B,HW,C1,C2,silu", [(2, 256, 320, 0, True), (2, 64, 1280, 1280, True),
                                             (3, 1024, 64, 0, False), (2, 16, 128, 64, True),
                                             (8, 4096, 320, 0, True)])
def test_groupnorm_fwd_bwd(cuda, B, HW, C1, C2, silu):
    from pcm_b200 import ops
    C = C1 + C2
    x1 = _rand((B, HW, C1), cuda, 1, 1.5, 0.3)
    x2 = _rand((B, HW, C2), cuda, 2, 0.7, -0.2) if C2 else None
    gamma = (torch.randn(C, device=cuda) * 0.2 + 1)
    beta = torch.randn(C, device=cuda) * 0.2
    out = torch.empty(B, HW, C, device=cuda, dtype=BF)
    stats = torch.empty(B, 32, 2, device=cuda)
    ops.groupnorm_fwd(x1, x2, gamma, beta, 1e-5, silu, out, stats, B, HW)
    xin = (torch.cat([x1, x2], -1) if C2 else x1).float().requires_grad_(True)
    y = F.group_norm(xin.transpose(1, 2), 32, gamma, beta, 1e-5)
    if silu:
        y = F.silu(y)
    ref = y.transpose(1, 2)
    _close(out, ref)
    dy = _rand((B, HW, C), cuda, 3)
    add = _rand((B, HW, C), cuda, 4)
    ref.backward(dy.float())
    gref = xin.grad + add.float()
    dx1 = torch.empty_like(x1)
    dx2 = torch.empty_like(x2) if C2 else None
    red = torch.empty(B, 32, 2, device=cuda)
    ops.groupnorm_bwd(dy, x1, x2, gamma, beta, 1e-5, silu, stats, red, add, dx1, dx2, B, HW)
    _close(dx1, gref[..., :C1], tol=2e-2)
    if C2:
        _close(dx2, gref[..., C1:], tol=2e-2)


@pytest.mark.parametrize("B,HW,C,shift,scale", [(2, 1024, 320, 60.0, 0.5), (2, 4096, 320, -200.0, 1.0),
                                                 (3, 256, 1280, 30.0, 0.25)])
def test_groupnorm_large_mean(cuda, B, HW, C, shift, scale):
    """|mean| >> sigma (pretrained SD1.5 activations have such outlier channels): a one-pass
    E[x^2] - mean^2 variance in fp32 loses the variance to cancellation; the pivot-shifted / Chan
    statistics must match torch's Welford-style group_norm, forward and backward, eps = 1e-6."""
    from pcm_b200 import ops
    x = _rand((B, HW, C), cuda, 5, scale, shift)
    gamma = torch.randn(C, device=cuda) * 0.2 + 1
    beta = torch.randn(C, device=cuda) * 0.2
    out = torch.empty(B, HW, C, device=cuda, dtype=BF)
    stats = torch.empty(B, 32, 2, device=cuda)
    ops.groupnorm_fwd(x, None, gamma, beta, 1e-6, False, out, stats, B, HW)
    xin = x.double().requires_grad_(True)
    ref = F.group_norm(xin.transpose(1, 2), 32, gamma.double(), beta.double(), 1e-6).transpose(1, 2)
    _close(out, ref)
    xg = xin.detach().view(B, HW, 32, C // 32)
    mean = xg.mean(dim=(1, 3))
    rstd = (xg.var(dim=(1, 3), unbiased=False) + 1e-6).rsqrt()
    assert torch.allclose(stats[..., 0].double(), mean, rtol=1e-5, atol=1e-5)
    assert torch.allclose(stats[..., 1].double(), rstd, rtol=2e-4), (stats[..., 1].double() / rstd - 1).abs().max()
    dy = _rand((B, HW, C), cuda, 6)
    ref.backward(dy.double())
    dx = torch.empty_like(x)
    red = torch.empty(B, 32, 2, device=cuda)
    ops.groupnorm_bwd(dy, x, None, gamma, beta, 1e-6, False, stats, red, None, dx, None, B, HW)
    _close(dx, xin.grad, tol=2e-2)


def test_groupnorm_reproducible_and_colsum(cuda):
    """Statistics, backward sums and per-image column sums are merged in block order: repeated
    launches are bit-identical; the column sums match a float64 reference."""
    from pcm_b200 import ops
    B, HW, C = 3, 1024, 640
    x = _rand((B, HW, C), cuda, 1, 1.5, 0.3)
    dy = _rand((B, HW, C), cuda, 3)
    gamma = torch.randn(C, device=cuda) * 0.2 + 1
    beta = torch.randn(C, device=cuda) * 0.2
    runs = []
    for _ in range(4):
        out = torch.empty(B, HW, C, device=cuda, dtype=BF)
        stats = torch.empty(B, 32, 2, device=cuda)
        ops.groupnorm_fwd(x, None, gamma, beta, 1e-5, True, out, stats, B, HW)
        dx = torch.empty_like(x)
        red = torch.empty(B, 32, 2, device=cuda)
        cs = torch.empty(B, C, device=cuda)
        ops.groupnorm_bwd(dy, x, None, gamma, beta, 1e-5, True, stats, red, None, dx, None, B, HW, colsum=cs)
        torch.cuda.synchronize()
        runs.append((out, stats, dx, red, cs))
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)
    dx, cs = runs[0][2], runs[0][4]
    # the kernel sums its unrounded fp32 dx; the bf16-rounded dx differs by rounding noise only
    assert torch.allclose(cs.double(), dx.double().sum(1), rtol=2e-2, atol=2e-2 * dx.double().sum(1).abs().max().item())


@pytest.mark.parametrize("M,C", [(1000, 320), (256, 1280), (77, 64), (512, 640)])
def test_layernorm_fwd_bwd(cuda, M, C):
    from pcm_b200 import ops
    x = _rand((M, C), cuda, 1, 2.0, 0.5)
    gamma = torch.randn(C, device=cuda) * 0.2 + 1
    beta = torch.randn(C, device=cuda) * 0.2
    out = torch.empty_like(x)
    stats = torch.empty(M, 2, device=cuda)
    ops.layernorm_fwd(x, gamma, beta, out, stats)
    xin = x.float().requires_grad_(True)
    ref = F.layer_norm(xin, (C,), gamma, beta, 1e-5)
    _close(out, ref)
    dy = _rand((M, C), cuda, 2)
    add = _rand((M, C), cuda, 3)
    ref.backward(dy.float())
    dx = torch.empty_like(x)
    ops.layernorm_bwd(dy, x, gamma, stats, add, dx)
    _close(dx, xin.grad + add.float(), tol=2e-2)


def test_geglu(cuda):
    from pcm_b200 import ops
    M, Fd = 500, 1280
    u = _rand((M, 2 * Fd), cuda, 1)
    out = torch.empty(M, Fd, device=cuda, dtype=BF)
    ops.geglu_fwd(u, out)
    uf = u.float().requires_grad_(True)
    a, g = uf.chunk(2, -1)
    ref = a * F.gelu(g)
    _close(out, ref)
    d = _rand((M, Fd), cuda, 2)
    ref.backward(d.float())
    du = torch.empty_like(u)
    ops.geglu_bwd(d, u, du)
    _close(du, uf.grad)


def test_upsample(cuda):
    from pcm_b200 import ops
    x = _rand((2, 8, 8, 64), cuda, 1)
    out = torch.empty(2, 16, 16, 64, device=cuda, dtype=BF)
    ops.upsample2x_fwd(x, out)
    xf = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    ref = F.interpolate(xf, scale_factor=2.0, mode="nearest")
    assert torch.equal(out.float().permute(0, 3, 1, 2), ref.detach())
    d = _rand((2, 16, 16, 64), cuda, 2)
    ref.backward(d.float().permute(0, 3, 1, 2))
    din = torch.empty_like(x)
    ops.upsample2x_bwd(d, din)
    _close(din.permute(0, 3, 1, 2), xf.grad)


def test_conv_c4_in_and_out_grad(cuda):
    from pcm_b200 import ops
    B, H, W, C = 2, 16, 16, 320
    x = torch.randn(B, H, W, 4, device=cuda)
    w = _rand((C, 4, 3, 3), cuda, 1, 0.2)
    bias = torch.randn(C, device=cuda)
    out = torch.empty(B, H, W, C, device=cuda, dtype=BF)
    ops.conv3x3_c4(x, w.permute(0, 2, 3, 1).contiguous(), bias, out, sgn=1, round_in=True)
    ref = F.conv2d(x.to(BF).float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    _close(out.permute(0, 3, 1, 2), ref)
    # conv_out (C -> 4) input gradient
    wo = _rand((4, C, 3, 3), cuda, 2, 0.05)
    dy = torch.randn(B, H, W, 4, device=cuda)
    xin = torch.zeros(B, C, H, W, device=cuda, requires_grad=True)
    F.conv2d(xin, wo.float(), padding=1).backward(dy.permute(0, 3, 1, 2))
    dx = torch.empty(B, H, W, C, device=cuda, dtype=BF)
    ops.conv3x3_c4(dy, wo.permute(1, 2, 3, 0).contiguous(), None, dx, sgn=-1, round_in=False)
    _close(dx.permute(0, 3, 1, 2), xin.grad)


def test_timestep_embed_colsum_add(cuda):
    from pcm_b200 import ops
    t = torch.tensor([0, 19, 499, 999], device=cuda)
    out = torch.empty(4, 320, device=cuda, dtype=BF)
    ops.timestep_embed(t, out)
    half = 160
    f = torch.exp(-math.log(10000.0) * torch.arange(half, device=cuda, dtype=torch.float32) / half)
    e = t[:, None].float() * f[None]
    ref = torch.cat([torch.cos(e), torch.sin(e)], -1)
    assert (out.float() - ref).abs().max().item() < 8e-3
    x = _rand((3, 100, 320), cuda, 1)
    cs = torch.empty(3, 320, device=cuda, dtype=BF)
    ops.colsum(x, cs, 3, 100)
    _close(cs, x.float().sum(1))
    a, b = _rand((1024,), cuda, 2), _rand((1024,), cuda, 3)
    o = torch.empty_like(a)
    ops.add_bf16(a, b, o)
    assert torch.equal(o, (a.float() + b.float()).to(BF))
