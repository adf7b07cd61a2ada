"""ORACLE (test infrastructure only -- never imported by the product path).

Plain-PyTorch CPU restatement of diffusers==0.26.3 ``AutoencoderKL`` as the reference calls it
(``vae.encode(pixels).latent_dist.sample() * scaling_factor``, train_pcm_lora_sd15.py:1127-1136, and the
validation pipeline's ``vae.decode``): ``Encoder`` (DownEncoderBlock2D with Downsample2D(padding=0): input
padded (0, 1, 0, 1), then a stride-2 convolution without padding), ``Decoder`` (UpDecoderBlock2D with nearest
2x Upsample2D), ``UNetMidBlock2D`` (ResnetBlock2D without temb, ``Attention(heads=1, residual_connection=True,
upcast_softmax=True, bias=True)``), ``DiagonalGaussianDistribution``, ``quant_conv`` / ``post_quant_conv``.
PARITY UNPINNED, as for unet_ref.py: diffusers is not installed here; the restatement is anchored by the
parameter inventory of the SD1.5 VAE (83,653,863 parameters: encoder with quant_conv 34,163,664, decoder
with post_quant_conv 49,490,199; tests/test_vae_cpu.py).

Parameters live in a flat dict keyed by diffusers state-dict names (``encoder.…``, ``decoder.…``,
``quant_conv.…``, ``post_quant_conv.…``; attention ``to_q / to_k / to_v / to_out.0``).

``emulate_bf16=True`` rounds weights and every tensor the CUDA path (pcm_b200/vae.py) materialises to bf16:
activations, GroupNorm outputs, q / k / v, the softmax probabilities, the attention output, the fp32 GEMM
outputs of conv_out and the moments.  The attention scores and the softmax statistics stay fp32.  The
network runs in the dtype of its parameters (float64 included).
"""
from dataclasses import dataclass
from typing import Dict, Tuple

import torch
import torch.nn.functional as F


@dataclass
class VAEConfig:
    in_channels: int = 3
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    latent_channels: int = 4
    norm_num_groups: int = 32
    scaling_factor: float = 0.18215


SD15 = VAEConfig()
SDXL = VAEConfig(scaling_factor=0.13025)
TINY = VAEConfig(block_out_channels=(64, 128), layers_per_block=1)


def layer_table(cfg: VAEConfig):
    """Ordered (name, kind, cin, cout, ksize) of every weight layer; kind "conv", "gn" or "linear"."""
    L = []
    ch = cfg.block_out_channels
    lat = cfg.latent_channels

    def resnet(p, cin, cout):
        L.append((p + ".norm1", "gn", cin, cin, 0))
        L.append((p + ".conv1", "conv", cin, cout, 3))
        L.append((p + ".norm2", "gn", cout, cout, 0))
        L.append((p + ".conv2", "conv", cout, cout, 3))
        if cin != cout:
            L.append((p + ".conv_shortcut", "conv", cin, cout, 1))

    def mid(p, c):
        resnet(p + ".resnets.0", c, c)
        a = p + ".attentions.0"
        L.append((a + ".group_norm", "gn", c, c, 0))
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            L.append((a + "." + n, "linear", c, c, 0))
        resnet(p + ".resnets.1", c, c)

    L.append(("encoder.conv_in", "conv", cfg.in_channels, ch[0], 3))
    cin = ch[0]
    for i, c in enumerate(ch):
        for j in range(cfg.layers_per_block):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", cin, c)
            cin = c
        if i < len(ch) - 1:
            L.append((f"encoder.down_blocks.{i}.downsamplers.0.conv", "conv", c, c, 3))
    mid("encoder.mid_block", ch[-1])
    L.append(("encoder.conv_norm_out", "gn", ch[-1], ch[-1], 0))
    L.append(("encoder.conv_out", "conv", ch[-1], 2 * lat, 3))
    L.append(("quant_conv", "conv", 2 * lat, 2 * lat, 1))
    L.append(("post_quant_conv", "conv", lat, lat, 1))
    L.append(("decoder.conv_in", "conv", lat, ch[-1], 3))
    mid("decoder.mid_block", ch[-1])
    rev = list(reversed(ch))
    prev = rev[0]
    for i, c in enumerate(rev):
        for j in range(cfg.layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
        prev = c
        if i < len(ch) - 1:
            L.append((f"decoder.up_blocks.{i}.upsamplers.0.conv", "conv", c, c, 3))
    L.append(("decoder.conv_norm_out", "gn", ch[0], ch[0], 0))
    L.append(("decoder.conv_out", "conv", ch[0], cfg.out_channels, 3))
    return L


def count_params(cfg: VAEConfig):
    """(encoder + quant_conv, decoder + post_quant_conv) parameter counts."""
    enc = dec = 0
    for name, kind, cin, cout, k in layer_table(cfg):
        n = 2 * cout if kind == "gn" else (cin * cout * (k * k if kind == "conv" else 1) + cout)
        if name.startswith(("encoder.", "quant_conv")):
            enc += n
        else:
            dec += n
    return enc, dec


def init_params(cfg: VAEConfig, seed: int = 0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights: nn.Conv2d / nn.Linear default init (U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for
    weight and bias); GroupNorm affine weights 1 + U(-0.1, 0.1), biases U(-0.1, 0.1) so that they matter."""
    g = torch.Generator().manual_seed(seed)
    P = {}

    def uni(shape, bound):
        return (torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1) * bound

    for name, kind, cin, cout, k in layer_table(cfg):
        if kind == "gn":
            P[name + ".weight"] = 1 + uni((cout,), 0.1)
            P[name + ".bias"] = uni((cout,), 0.1)
        elif kind == "conv":
            P[name + ".weight"] = uni((cout, cin, k, k), (cin * k * k) ** -0.5)
            P[name + ".bias"] = uni((cout,), (cin * k * k) ** -0.5)
        else:
            P[name + ".weight"] = uni((cout, cin), cin ** -0.5)
            P[name + ".bias"] = uni((cout,), cin ** -0.5)
    return {k: v.to(dtype) for k, v in P.items()}


class VAERef:
    """Functional AutoencoderKL over a flat parameter dict (NCHW tensors)."""

    def __init__(self, cfg: VAEConfig, P, emulate_bf16=False):
        self.cfg, self.emu = cfg, emulate_bf16
        self.P = {k: self._q(v) for k, v in P.items()} if emulate_bf16 else P

    def _q(self, x):
        return x.to(torch.bfloat16).to(x.dtype) if self.emu else x

    def conv(self, name, x, stride=1, padding=1, residual=None):
        W, b = self.P[name + ".weight"], self.P[name + ".bias"]
        y = F.conv2d(x, W, b, stride=stride, padding=padding if W.shape[-1] == 3 else 0)
        if residual is not None:
            y = y + residual
        return self._q(y)

    def gn(self, name, x, silu):
        y = F.group_norm(x, self.cfg.norm_num_groups, self.P[name + ".weight"], self.P[name + ".bias"], 1e-6)
        return self._q(F.silu(y) if silu else y)

    def resnet(self, p, x):
        h = self.gn(p + ".norm1", x, True)
        h = self.conv(p + ".conv1", h)
        h = self.gn(p + ".norm2", h, True)
        sc = self.conv(p + ".conv_shortcut", x) if (p + ".conv_shortcut.weight") in self.P else x
        return self.conv(p + ".conv2", h, residual=sc)

    def attention(self, p, x):
        B, C, H, W = x.shape
        h = self.gn(p + ".group_norm", x, False).flatten(2).transpose(1, 2)      # [B, HW, C]

        def lin(n, t, residual=None):
            y = F.linear(t, self.P[f"{p}.{n}.weight"], self.P[f"{p}.{n}.bias"])
            return self._q(y if residual is None else y + residual)

        q, k, v = lin("to_q", h), lin("to_k", h), lin("to_v", h)
        s = (q @ k.transpose(1, 2)) * C ** -0.5
        a = self._q(torch.softmax(s, -1))
        o = self._q(a @ v)
        return lin("to_out.0", o, x.flatten(2).transpose(1, 2)).transpose(1, 2).reshape(B, C, H, W)

    def mid(self, p, x):
        x = self.resnet(p + ".resnets.0", x)
        x = self.attention(p + ".attentions.0", x)
        return self.resnet(p + ".resnets.1", x)

    def encode(self, images):
        """images NCHW in [-1, 1] -> (mean, logvar) of the latent distribution, logvar clamped."""
        cfg = self.cfg
        x = self.conv("encoder.conv_in", self._q(images))
        for i in range(len(cfg.block_out_channels)):
            for j in range(cfg.layers_per_block):
                x = self.resnet(f"encoder.down_blocks.{i}.resnets.{j}", x)
            if i < len(cfg.block_out_channels) - 1:
                x = self.conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", F.pad(x, (0, 1, 0, 1)), stride=2,
                              padding=0)
        x = self.mid("encoder.mid_block", x)
        x = self.gn("encoder.conv_norm_out", x, True)
        x = self.conv("encoder.conv_out", x)
        m = self.conv("quant_conv", x)
        mean, logvar = m.chunk(2, dim=1)
        return mean, logvar.clamp(-30.0, 20.0)

    def decode(self, z):
        """z NCHW latents (already divided by the scaling factor) -> NCHW image in about [-1, 1]."""
        cfg = self.cfg
        x = self.conv("post_quant_conv", self._q(z))
        x = self.conv("decoder.conv_in", x)
        x = self.mid("decoder.mid_block", x)
        n = len(cfg.block_out_channels)
        for i in range(n):
            for j in range(cfg.layers_per_block + 1):
                x = self.resnet(f"decoder.up_blocks.{i}.resnets.{j}", x)
            if i < n - 1:
                x = self.conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", F.interpolate(x, scale_factor=2.0,
                                                                                         mode="nearest"))
        x = self.gn("decoder.conv_norm_out", x, True)
        return self.conv("decoder.conv_out", x)


def sample(mean, logvar, noise):
    """DiagonalGaussianDistribution.sample with the caller's noise: mean + exp(logvar / 2) * noise."""
    return mean + torch.exp(0.5 * logvar) * noise
