"""Test-side torch semantics of the VAE's `pcm_b200.ops` wrappers (include/pcm_b200.h), on top of
ops_interp.install: with install(monkeypatch) the host code of pcm_b200/vae.py runs on CPU with every kernel
interpreted.  The GPU tests (tests/test_vae_gpu.py) check the CUDA kernels against the same statements."""
import torch

import gemm_interp
import ops_interp
from pcm_b200 import ops

BF16 = torch.bfloat16


def softmax_rows(s, p):
    p.copy_(torch.softmax(s.float(), -1).to(BF16))
    return p


def transpose_bf16(x, out):
    out.copy_(x.transpose(1, 2))
    return out


def latent_dist(h, w, bias, noise, scale, mean, logvar, std, sample):
    B, hh, ww, _ = h.shape
    m = (h.to(BF16).float().reshape(-1, 8) @ w.float().t() + bias).to(BF16).float()
    m = m.view(B, hh, ww, 8).permute(0, 3, 1, 2)
    mean.copy_(m[:, :4])
    logvar.copy_(m[:, 4:].clamp(-30.0, 20.0))
    std.copy_(torch.exp(0.5 * logvar))
    if noise is not None:
        sample.copy_((mean + std * noise) * scale)


def vae_dec_in(z, w, bias, div, out):
    x = (z / div).to(BF16).float().reshape(-1, 4)
    out.zero_()
    out[..., :4].copy_((x @ w.float().t() + bias).to(BF16).view(out[..., :4].shape))
    return out


def gemm(a_srcs, b_srcs, prog, **kw):
    """gemm_interp.interp_gemm, also for entries whose operands end inside their 64-wide chunk (the decoder's
    conv_in: 8-channel pixels, 8-column taps): the kernel multiplies the columns both operands have, rounded up
    to 16, against TMA-filled zeros, which is the product of the operands zero-padded to whole chunks."""
    keep, a_srcs, b_srcs = [], list(a_srcs), list(b_srcs)
    for e in prog:
        a, b = a_srcs[e[0]], b_srcs[e[1]]
        if a.C < e[5] + 64 * e[4]:
            x = gemm_interp.a_nhwc(a)
            x = torch.cat([x, x.new_zeros(*x.shape[:3], e[5] + 64 * e[4] - a.C)], -1)
            keep.append(x)
            a_srcs[e[0]] = ops.asrc_nhwc(x)
        if b.K < e[6] + 64 * e[4]:
            w = gemm_interp.b_matrix(b)
            w = torch.cat([w, w.new_zeros(w.shape[0], e[6] + 64 * e[4] - b.K)], -1)
            keep.append(w)
            b_srcs[e[1]] = ops.bsrc(w)
    return gemm_interp.interp_gemm(a_srcs, b_srcs, prog, **kw)


def image_exit(x, out, u8=None):
    v = (x / 2 + 0.5).clamp(0, 1)
    if out is not None:
        out.copy_(v.permute(0, 3, 1, 2))
    if u8 is not None:
        u8.copy_((v * 255).round().to(torch.uint8))
    return out


def install(monkeypatch):
    ops_interp.install(monkeypatch)
    monkeypatch.setattr(ops, "gemm", gemm)
    for name in ("softmax_rows", "transpose_bf16", "latent_dist", "vae_dec_in", "image_exit"):
        monkeypatch.setattr(ops, name, globals()[name])
