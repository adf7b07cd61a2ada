"""The Stable Diffusion VAE (diffusers' AutoencoderKL) on the CUDA path, inference only.

What the reference runs around the UNet: `vae.encode(pixels).latent_dist.sample() * scaling_factor` for every
training batch (train_pcm_lora_sd15.py:1127-1136) and `vae.decode(latents / scaling_factor)` in the
validation pipeline (log_validation).  Python only sequences C-ABI launches (pcm_b200.ops):
  * activations NHWC bf16, one rounding per materialised tensor (bf16 autocast semantics);
  * every 3x3 / 1x1 convolution and Linear layer is the wgmma implicit GEMM (UNet K programs, unet.conv_prog),
    GroupNorm(+SiLU) the UNet's kernels, the shortcut / attention residual enters the GEMM epilogue;
  * Downsample2D(padding=0): the input padded by (0, 1, 0, 1) and a stride-2 convolution without padding is
    the parity-plane program with its own tap table (_S2_VAE); TMA zero fill past the plane is the padding;
  * the mid-block attention (1 head, d = C) runs as GEMMs: q / k / v in one launch, then per image and per
    chunk of query rows S = d^-1/2 Q K^T (fp32), P = softmax(S) (pcm_softmax_rows, bf16), O = P V with
    V^T from pcm_transpose_bf16; to_out adds the residual in its epilogue;
  * the encoder's conv_in: pcm_conv3x3_c4 (RGB padded to a zero fourth channel); the decoder's conv_in (4 -> 512
    channels, more than pcm_conv3x3_c4 holds): pcm_vae_dec_in (post_quant_conv) writes bf16 pixels of 8 channels,
    4 of them zero, and the implicit GEMM runs the 3x3 convolution as 9 taps of one 8-wide K chunk each;
    quant_conv and the latent distribution: pcm_latent_dist; the image exit (x / 2 + 0.5).clamp(0, 1):
    pcm_image_exit.
Image widths: at every resolution level the width must divide 128 or be a multiple of 128 (512 and 1024 pixel
images, and any image of at most 128 pixels per side that halves evenly).
"""
import json
import os
import types
from dataclasses import dataclass
from typing import Tuple

import torch

from . import ops
from .unet import TAPS3, conv_prog

BF16 = torch.bfloat16
# Downsample2D(padding=0) after F.pad(x, (0, 1, 0, 1)): kernel index -> (input parity, shift in the parity
# plane): 0 -> plane 0, 0; 1 -> plane 1, 0; 2 -> plane 0, +1 (the row past the last is the zero padding)
_S2_VAE = ((0, 0), (1, 0), (0, 1))
# largest activation of one launch, in elements: decoding 16 images at 512^2 (256 channels at full resolution)
# reaches exactly this; bigger batches run in sub-batches (tests/test_vae_gpu.py proves a GEMM of this size)
MAX_LAUNCH_ELEMENTS = 1 << 30
# fp32 attention scores of one chunk of query rows: at most this many elements (128 MB, plus 64 MB of bf16 P)
_ATTN_CHUNK_ELEMENTS = 1 << 25
_LEGACY_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


@dataclass
class VAEConfig:
    in_channels: int = 3
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    latent_channels: int = 4
    norm_num_groups: int = 32
    scaling_factor: float = 0.18215

    @classmethod
    def from_dict(cls, d):
        kw = {k: d[k] for k in ("in_channels", "out_channels", "layers_per_block", "latent_channels",
                                 "norm_num_groups", "scaling_factor") if k in d}
        if "block_out_channels" in d:
            kw["block_out_channels"] = tuple(d["block_out_channels"])
        cfg = cls(**kw)
        if cfg.in_channels != 3 or cfg.out_channels != 3 or cfg.latent_channels != 4:
            raise ValueError("the CUDA VAE runs 3-channel images and 4 latent channels")
        if any(c % 64 for c in cfg.block_out_channels) or any(c % cfg.norm_num_groups for c in cfg.block_out_channels):
            raise ValueError(f"block_out_channels {cfg.block_out_channels}: each must be a multiple of 64 and of "
                             f"norm_num_groups {cfg.norm_num_groups}")
        if cfg.block_out_channels[0] > 320:
            raise ValueError("the encoder's conv_in (pcm_conv3x3_c4) takes at most 320 channels")
        return cfg


def layer_table(cfg: VAEConfig):
    """Ordered (name, kind, cin, cout, ksize) of every weight layer, diffusers names; kind conv / gn / linear."""
    L, ch, lat = [], cfg.block_out_channels, cfg.latent_channels

    def resnet(p, cin, cout):
        L.extend([(p + ".norm1", "gn", cin, cin, 0), (p + ".conv1", "conv", cin, cout, 3),
                  (p + ".norm2", "gn", cout, cout, 0), (p + ".conv2", "conv", cout, cout, 3)])
        if cin != cout:
            L.append((p + ".conv_shortcut", "conv", cin, cout, 1))

    def mid(p, c):
        resnet(p + ".resnets.0", c, c)
        L.append((p + ".attentions.0.group_norm", "gn", c, c, 0))
        L.extend((f"{p}.attentions.0.{n}", "linear", c, c, 0) for n in ("to_q", "to_k", "to_v", "to_out.0"))
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
    L += [("encoder.conv_norm_out", "gn", ch[-1], ch[-1], 0), ("encoder.conv_out", "conv", ch[-1], 2 * lat, 3),
          ("quant_conv", "conv", 2 * lat, 2 * lat, 1), ("post_quant_conv", "conv", lat, lat, 1),
          ("decoder.conv_in", "conv", lat, ch[-1], 3)]
    mid("decoder.mid_block", ch[-1])
    rev = list(reversed(ch))
    prev = rev[0]
    for i, c in enumerate(rev):
        for j in range(cfg.layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
        prev = c
        if i < len(ch) - 1:
            L.append((f"decoder.up_blocks.{i}.upsamplers.0.conv", "conv", c, c, 3))
    L += [("decoder.conv_norm_out", "gn", ch[0], ch[0], 0), ("decoder.conv_out", "conv", ch[0], cfg.out_channels, 3)]
    return L


def synthetic_state_dict(cfg: VAEConfig, seed=0):
    """Seeded random weights (nn.Conv2d / nn.Linear default init; GroupNorm affine 1 + U(-0.1, 0.1), U(-0.1, 0.1))."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def uni(shape, bound):
        return (torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1) * bound

    for name, kind, cin, cout, k in layer_table(cfg):
        if kind == "gn":
            sd[name + ".weight"], sd[name + ".bias"] = 1 + uni((cout,), 0.1), uni((cout,), 0.1)
        elif kind == "conv":
            sd[name + ".weight"] = uni((cout, cin, k, k), (cin * k * k) ** -0.5)
            sd[name + ".bias"] = uni((cout,), (cin * k * k) ** -0.5)
        else:
            sd[name + ".weight"], sd[name + ".bias"] = uni((cout, cin), cin ** -0.5), uni((cout,), cin ** -0.5)
    return sd


def canonical_state_dict(sd):
    """diffusers key names: the legacy attention spelling query / key / value / proj_attn becomes
    to_q / to_k / to_v / to_out.0 (1x1-convolution shaped attention weights become [C, C])."""
    out = {}
    for k, v in sd.items():
        parts = k.split(".")
        if ".attentions." in k and parts[-2] in _LEGACY_ATTN:
            k = ".".join(parts[:-2] + [_LEGACY_ATTN[parts[-2]], parts[-1]])
        if ".attentions." in k and k.endswith(".weight") and v.dim() == 4:
            v = v.reshape(v.shape[0], v.shape[1])
        out[k] = v
    return out


class DiagonalGaussianDistribution:
    """The encoder's latent distribution, fp32 NCHW [B, 4, h, w]: .mean, .logvar (clamped to [-30, 20]), .std."""

    def __init__(self, vae, h, mean, logvar, std):
        self._vae, self._h = vae, h
        self.mean, self.logvar, self.std = mean, logvar, std

    def sample(self, generator=None):
        """mean + std * noise, noise = randn(B, 4, h, w, generator) (diffusers' randn_tensor order), fp32."""
        gdev = generator.device if generator is not None else self.mean.device
        noise = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=torch.float32)
        noise = noise.to(self.mean.device)
        out = torch.empty_like(self.mean)
        v = self._vae
        ops.latent_dist(self._h, v.quant_w, v.quant_b, noise, 1.0, torch.empty_like(self.mean),
                        torch.empty_like(self.mean), torch.empty_like(self.mean), out)
        return out

    def mode(self):
        return self.mean


class AutoencoderKL:
    """vae = AutoencoderKL.from_pretrained("runwayml/stable-diffusion-v1-5" path, subfolder="vae")
    latents = vae.encode(images).latent_dist.sample(generator) * vae.config.scaling_factor
    images = vae.decode(latents / vae.config.scaling_factor).sample
    CUDA tensors only; images NCHW fp32 in [-1, 1]."""

    def __init__(self, cfg: VAEConfig, state_dict, device="cuda"):
        self.cfg, self.config, self.dev = cfg, cfg, device
        sd = canonical_state_dict(state_dict)
        self.layers = {}
        for name, kind, cin, cout, k in layer_table(cfg):
            L = types.SimpleNamespace(name=name, kind=kind, cin=cin, cout=cout, k=k)
            W = sd[name + ".weight"].float()
            b = sd[name + ".bias"].float()
            if tuple(W.shape) != ((cout,) if kind == "gn" else (cout, cin, k, k) if kind == "conv" else (cout, cin)):
                raise ValueError(f"{name}.weight: shape {tuple(W.shape)} does not match the config")
            L.bias = b.to(device)
            if kind == "gn":
                L.gamma, L.beta = W.to(device), L.bias
            elif name == "encoder.conv_in":                              # pcm_conv3x3_c4: [C][3][3][4]
                w4 = torch.zeros(cout, 3, 3, 4)
                w4[..., :cin] = W.permute(0, 2, 3, 1)
                L.w_c4 = w4.to(device=device, dtype=BF16)
            elif name == "decoder.conv_in":                              # [N, 9 taps x 8 channels], 4 of them 0
                w8 = torch.zeros(cout, 3, 3, 8)
                w8[..., :cin] = W.permute(0, 2, 3, 1)
                L.w = w8.reshape(cout, 72).to(device=device, dtype=BF16).contiguous()
            elif name in ("quant_conv", "post_quant_conv"):
                L.w = W.reshape(cout, cin).to(device=device, dtype=BF16).contiguous()
            elif kind == "conv":                                            # [N, taps * cin], K-blocked
                L.w = ops.kblock(W.permute(0, 2, 3, 1).reshape(cout, -1).to(device=device, dtype=BF16))
            self.layers[name] = L
        for p in ("encoder.mid_block.attentions.0", "decoder.mid_block.attentions.0"):   # q / k / v as ONE GEMM
            A = types.SimpleNamespace(C=self.layers[p + ".to_q"].cin)
            A.w_qkv = ops.kblock(torch.cat([sd[f"{p}.{n}.weight"].float() for n in ("to_q", "to_k", "to_v")])
                                 .reshape(3 * A.C, A.C).to(device=device, dtype=BF16))
            A.b_qkv = torch.cat([self.layers[f"{p}.{n}"].bias for n in ("to_q", "to_k", "to_v")]).contiguous()
            A.w_out = ops.kblock(sd[p + ".to_out.0.weight"].float().reshape(A.C, A.C).to(device=device, dtype=BF16))
            A.b_out = self.layers[p + ".to_out.0"].bias
            self.layers[p] = A
        self.quant_w, self.quant_b = self.layers["quant_conv"].w, self.layers["quant_conv"].bias
        self.held = []      # GroupNorm workspaces captured graphs may point at

    @classmethod
    def from_pretrained(cls, path=None, subfolder="vae", device="cuda", config=None, seed=0):
        """`path`/`subfolder`: config.json and diffusion_pytorch_model.safetensors (diffusers layout).  path=None:
        a seeded random network of `config` (default SD1.5's)."""
        if path is None:
            cfg = config if isinstance(config, VAEConfig) else VAEConfig.from_dict(config or {})
            return cls(cfg, synthetic_state_dict(cfg, seed), device)
        from safetensors.torch import load_file
        d = os.path.join(path, subfolder) if subfolder else path
        with open(os.path.join(d, "config.json")) as f:
            cfg = VAEConfig.from_dict(json.load(f))
        return cls(cfg, load_file(os.path.join(d, "diffusion_pytorch_model.safetensors")), device)

    # ------------------------------------------------------------------------------------------
    def _new(self, *shape, dtype=BF16):
        return torch.empty(*shape, device=self.dev, dtype=dtype)

    def conv(self, name, x, stride=1, residual=None, out_fp32=False):
        """3x3 (pad 1, or stride 2 after the (0, 1, 0, 1) pad) or 1x1 convolution of NHWC x, bias (+ residual) in
        the epilogue."""
        L = self.layers[name]
        B, H, W, _ = x.shape
        Ho, Wo = H // stride, W // stride
        M, N = B * Ho * Wo, L.cout
        out = self._new(B, Ho, Wo, N, dtype=torch.float32 if out_fp32 else BF16)
        res = None if residual is None else residual.reshape(M, N)
        if L.k == 1:
            ops.gemm([ops.asrc_mat(x.view(M, L.cin))], [ops.bsrc(L.w)], [(0, 0, 0, 0, L.cin // 64, 0, 0)], lin=True,
                     M=M, N=N, out=out.view(M, N), bias=L.bias, residual=res)
            return out
        srcs, prog = conv_prog([x], 3, stride, L.cin, _S2_VAE)
        ops.gemm(srcs, [ops.bsrc(L.w)], prog, lin=False, M=M, N=N, geo=(Wo, Ho), out=out.view(M, N), bias=L.bias,
                 residual=res, round_bf16=out_fp32)
        return out

    def gn(self, name, x, silu):
        L = self.layers[name]
        B, H, W, C = x.shape
        out = self._new(B, H, W, C)
        stats = self._new(B, self.cfg.norm_num_groups, 2, dtype=torch.float32)
        ops.groupnorm_fwd(x.view(B * H * W, C), None, L.gamma, L.beta, 1e-6, silu, out.view(B * H * W, C), stats,
                          B, H * W, self.cfg.norm_num_groups)
        return out

    def resnet(self, p, x):
        """ResnetBlock2D without temb: GN+SiLU, conv1, GN+SiLU, conv2 + shortcut (1x1 where cin != cout)."""
        h = self.gn(p + ".norm1", x, True)
        h = self.conv(p + ".conv1", h)
        h = self.gn(p + ".norm2", h, True)
        sc = self.conv(p + ".conv_shortcut", x) if (p + ".conv_shortcut") in self.layers else x
        return self.conv(p + ".conv2", h, residual=sc)

    def attention(self, p, x):
        """Attention(heads=1, d = C, residual_connection, upcast_softmax) over the H*W tokens of each image."""
        A = self.layers[p]
        B, H, W, C = x.shape
        S, M = H * W, B * H * W
        if S % 8:
            raise ValueError(f"mid-block attention needs a multiple of 8 tokens, got {S}")
        g = self.gn(p + ".group_norm", x, False).view(M, C)
        qkv = self._new(M, 3 * C)
        ops.gemm([ops.asrc_mat(g)], [ops.bsrc(A.w_qkv)], [(0, 0, 0, 0, C // 64, 0, 0)], lin=True, M=M, N=3 * C,
                 out=qkv, bias=A.b_qkv)
        vt = self._new(B, C, S)
        ops.transpose_bf16(qkv.view(B, S, 3 * C)[:, :, 2 * C:], vt)
        R = min(S, max(128, _ATTN_CHUNK_ELEMENTS // S // 128 * 128))
        s32 = self._new(R, S, dtype=torch.float32)
        pr = self._new(R, S)
        o = self._new(M, C)
        for b in range(B):
            k = qkv[b * S:(b + 1) * S, C:2 * C]
            for r0 in range(0, S, R):
                r = min(R, S - r0)
                rows = slice(b * S + r0, b * S + r0 + r)
                ops.gemm([ops.asrc_mat(qkv[rows, :C])], [ops.bsrc(k)], [(0, 0, 0, 0, C // 64, 0, 0)], lin=True,
                         M=r, N=S, out=s32[:r], alpha=C ** -0.5)
                ops.softmax_rows(s32[:r], pr[:r])
                ops.gemm([ops.asrc_mat(pr[:r])], [ops.bsrc(vt[b])], [(0, 0, 0, 0, (S + 63) // 64, 0, 0)], lin=True,
                         M=r, N=C, out=o[rows])
        out = self._new(B, H, W, C)
        ops.gemm([ops.asrc_mat(o)], [ops.bsrc(A.w_out)], [(0, 0, 0, 0, C // 64, 0, 0)], lin=True, M=M, N=C,
                 out=out.view(M, C), bias=A.b_out, residual=x.reshape(M, C))
        return out

    def mid(self, p, x):
        x = self.resnet(p + ".resnets.0", x)
        x = self.attention(p + ".attentions.0", x)
        return self.resnet(p + ".resnets.1", x)

    # ------------------------------------------------------------------------------------------
    def _check_size(self, H, W, what):
        n = len(self.cfg.block_out_channels)
        for lv in range(n):
            h, w = H >> lv, W >> lv
            if (h << lv) != H or (w << lv) != W or not (128 % w == 0 or w % 128 == 0):
                raise ValueError(f"{what}: {H}x{W} pixels; every level's width (here {w}) must divide 128 or be a "
                                 f"multiple of 128, and the size must halve {n - 1} times")

    def _per_pass(self, H, W):
        """Images per sub-batch: the largest activation (full resolution, max(C0, C1) channels) of one launch
        stays within MAX_LAUNCH_ELEMENTS."""
        per_image = H * W * max(self.cfg.block_out_channels[:2])
        return max(1, MAX_LAUNCH_ELEMENTS // per_image)

    def encode_nhwc(self, x4):
        """x4: fp32 NHWC [B, H, W, 4] images in [-1, 1] with a zero fourth channel -> h fp32 NHWC [B, h, w, 8]
        (encoder.conv_out, values rounded to bf16)."""
        cfg, ch = self.cfg, self.cfg.block_out_channels
        B, H, W, _ = x4.shape
        x = self._new(B, H, W, ch[0])
        L = self.layers["encoder.conv_in"]
        ops.conv3x3_c4(x4, L.w_c4, L.bias, x, sgn=1, round_in=True)
        for i in range(len(ch)):
            for j in range(cfg.layers_per_block):
                x = self.resnet(f"encoder.down_blocks.{i}.resnets.{j}", x)
            if i < len(ch) - 1:
                x = self.conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", x, stride=2)
        x = self.mid("encoder.mid_block", x)
        x = self.gn("encoder.conv_norm_out", x, True)
        return self.conv("encoder.conv_out", x, out_fp32=True)

    def decode_nhwc(self, z, div=1.0):
        """z: fp32 NHWC [B, h, w, 4] latents, divided by `div` on the way in -> fp32 NHWC [B, 8h, 8w, 3] (values
        rounded to bf16)."""
        cfg = self.cfg
        n = len(cfg.block_out_channels)
        B, h, w, _ = z.shape
        zin = self._new(B, h, w, 8)
        Lp = self.layers["post_quant_conv"]
        ops.vae_dec_in(z, Lp.w, Lp.bias, div, zin)
        L = self.layers["decoder.conv_in"]
        M = B * h * w
        x = self._new(B, h, w, L.cout)
        ops.gemm([ops.asrc_nhwc(zin)], [ops.bsrc(L.w)], [(0, 0, dw, dh, 1, 0, 8 * t) for t, (dw, dh) in enumerate(TAPS3)],
                 lin=False, M=M, N=L.cout, geo=(w, h), out=x.view(M, L.cout), bias=L.bias)
        x = self.mid("decoder.mid_block", x)
        for i in range(n):
            for j in range(cfg.layers_per_block + 1):
                x = self.resnet(f"decoder.up_blocks.{i}.resnets.{j}", x)
            if i < n - 1:
                Bx, Hx, Wx, Cx = x.shape
                xu = self._new(Bx, 2 * Hx, 2 * Wx, Cx)
                ops.upsample2x_fwd(x, xu)
                x = self.conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", xu)
        x = self.gn("decoder.conv_norm_out", x, True)
        return self.conv("decoder.conv_out", x, out_fp32=True)

    def _hold_workspaces(self):
        ws = ops._GN_WS.get(torch.device(self.dev))
        if ws is not None and all(ws is not h for h in self.held):
            self.held.append(ws)

    def encode(self, images):
        """images: NCHW fp32 in [-1, 1] -> .latent_dist (DiagonalGaussianDistribution)."""
        if not torch.is_tensor(images) or images.dim() != 4 or images.shape[1] != self.cfg.in_channels:
            raise ValueError(f"images must be [B, {self.cfg.in_channels}, H, W]")
        B, _, H, W = images.shape
        self._check_size(H, W, "encode")
        x4 = torch.zeros(B, H, W, 4, device=self.dev, dtype=torch.float32)
        x4[..., :3] = images.to(self.dev, torch.float32).permute(0, 2, 3, 1)
        n = len(self.cfg.block_out_channels) - 1
        step = self._per_pass(H, W)
        h = torch.cat([self.encode_nhwc(x4[i:i + step]) for i in range(0, B, step)]) if B > step else self.encode_nhwc(x4)
        self._hold_workspaces()
        mean, logvar, std = (self._new(B, 4, H >> n, W >> n, dtype=torch.float32) for _ in range(3))
        ops.latent_dist(h, self.quant_w, self.quant_b, None, 1.0, mean, logvar, std, None)
        return types.SimpleNamespace(latent_dist=DiagonalGaussianDistribution(self, h, mean, logvar, std))

    def decode(self, latents):
        """latents: NCHW fp32 [B, 4, h, w] (already divided by the scaling factor) -> .sample NCHW fp32."""
        if not torch.is_tensor(latents) or latents.dim() != 4 or latents.shape[1] != self.cfg.latent_channels:
            raise ValueError(f"latents must be [B, {self.cfg.latent_channels}, h, w]")
        n = len(self.cfg.block_out_channels) - 1
        B, _, h, w = latents.shape
        self._check_size(h << n, w << n, "decode")
        z = latents.to(self.dev, torch.float32).permute(0, 2, 3, 1).contiguous()
        step = self._per_pass(h << n, w << n)
        x = torch.cat([self.decode_nhwc(z[i:i + step]) for i in range(0, B, step)]) if B > step else self.decode_nhwc(z)
        self._hold_workspaces()
        return types.SimpleNamespace(sample=x.permute(0, 3, 1, 2).contiguous())

    def decode_images(self, z, div, out=None, u8=None):
        """The pipeline's decode + postprocess on NHWC latents z: (decode(z / div) / 2 + 0.5).clamp(0, 1) into
        out (fp32 NCHW) and u8 (uint8 NHWC, round(255 v)); sub-batched like decode()."""
        n = len(self.cfg.block_out_channels) - 1
        B, h, w, _ = z.shape
        self._check_size(h << n, w << n, "decode")
        step = self._per_pass(h << n, w << n)
        for i in range(0, B, step):
            x = self.decode_nhwc(z[i:i + step], div)
            ops.image_exit(x, None if out is None else out[i:i + step], None if u8 is None else u8[i:i + step])
        return out
