"""ORACLE (test infrastructure only -- never imported by the product path).

Plain-PyTorch CPU restatement of the third-party modules the reference's hot path calls:
  * diffusers==0.26.3 ``UNet2DConditionModel`` in the runwayml/stable-diffusion-v1-5 configuration
    (call sites: code/text_to_image_sd15/train_pcm_lora_sd15.py:1192-1198 student,
    :1219-1223 / :1238-1244 teacher, :1263-1268 target; construction :840, :849), and
  * peft==0.9.0 LoRA wrappers (train_pcm_lora_sd15.py:866-885: r=lora_rank, lora_alpha=8 default,
    14 target-module suffixes, A kaiming-uniform / B zeros).
Neither package is vendored in the reference repository nor installed in this environment (pinned in
code/text_to_image_sd15/environment.yaml:40,87), so the published semantics are restated from
SURVEY.md Appendix A (A2: UNet, A3: LoRA).  PARITY UNPINNED for the UNet itself: the reference
ships no golden vectors or tests for it; the PCM math around it is pinned separately
(oracle/pcm_ref.py vs the reference's own functions).

Parameters live in a flat dict keyed by diffusers state-dict names; LoRA tensors use
``<module path>.lora_A.weight`` / ``.lora_B.weight`` (peft's names minus the ``base_model.model.``
prefix and ``.default`` infix).

``emulate_bf16=True`` rounds weights and every tensor the CUDA path materialises in HBM to bf16
(straight-through in autograd); this mirrors the reference running under bf16 autocast.
``round_grads=True`` (with emulate_bf16) also rounds, in the backward, the gradient of every tensor whose
gradient the CUDA backward stores in bf16 (see UNetRef).

The network runs on the device and in the dtype of its parameters (float64 on CUDA included).
"""
import math
from dataclasses import dataclass
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

LORA_TARGETS = ("to_q", "to_k", "to_v", "to_out.0", "proj_in", "proj_out", "ff.net.0.proj",
                "ff.net.2", "conv1", "conv2", "conv_shortcut", "downsamplers.0.conv",
                "upsamplers.0.conv", "time_emb_proj")  # train_pcm_lora_sd15.py:868-883


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    cross_attention_dim: int = 768
    num_heads: int = 8            # SD1.5 `attention_head_dim=8` is interpreted as head COUNT
    norm_num_groups: int = 32
    # which down blocks carry attention (CrossAttnDownBlock2D x3, DownBlock2D)
    down_attn: Tuple[bool, ...] = (True, True, True, False)
    lora_rank: int = 64
    lora_alpha: float = 8.0       # peft LoraConfig default
    # SDXL-style extensions (diffusers config of stabilityai/stable-diffusion-xl-base-1.0; call sites
    # train_pcm_lora_sdxl_adv.py:1094-1133 added_cond_kwargs, :1215-1221 zero uncond embeddings)
    transformer_layers_per_block: Tuple[int, ...] = ()      # () -> 1 everywhere
    heads_per_block: Tuple[int, ...] = ()                   # () -> num_heads everywhere
    use_linear_projection: bool = False
    addition_embed: bool = False                            # addition_embed_type == "text_time"
    addition_time_embed_dim: int = 256
    text_embed_dim: int = 1280
    num_time_ids: int = 6

    def depth(self, level):
        return self.transformer_layers_per_block[level] if self.transformer_layers_per_block else 1

    def heads(self, level):
        return self.heads_per_block[level] if self.heads_per_block else self.num_heads

    @property
    def add_embed_in(self):
        return self.text_embed_dim + self.num_time_ids * self.addition_time_embed_dim

    @property
    def time_embed_dim(self):
        return self.block_out_channels[0] * 4

    @property
    def up_attn(self):
        return tuple(reversed(self.down_attn))


SD15 = UNetConfig()
TINY = UNetConfig(block_out_channels=(64, 128, 128, 128), cross_attention_dim=64, num_heads=2,
                  lora_rank=64)
SDXL = UNetConfig(block_out_channels=(320, 640, 1280), down_attn=(False, True, True),
                  transformer_layers_per_block=(1, 2, 10), heads_per_block=(5, 10, 20),
                  cross_attention_dim=2048, use_linear_projection=True, addition_embed=True)
TINY_XL = UNetConfig(block_out_channels=(64, 128, 128), down_attn=(False, True, True),
                     transformer_layers_per_block=(1, 2, 3), heads_per_block=(1, 2, 2),
                     cross_attention_dim=128, use_linear_projection=True, addition_embed=True,
                     addition_time_embed_dim=64, text_embed_dim=128)


# ---------------------------------------------------------------------------------------------
# parameter construction (seeded synthetic weights: PyTorch default nn.Conv2d / nn.Linear init)
# ---------------------------------------------------------------------------------------------
def _is_lora_target(name):
    return any(name == t or name.endswith("." + t) for t in LORA_TARGETS)


def layer_table(cfg: UNetConfig):
    """Ordered list of (name, kind, cin, cout, ksize) for every weight layer of the UNet."""
    L = []
    ch = cfg.block_out_channels
    temb = cfg.time_embed_dim

    def resnet(p, cin, cout):
        L.append((p + ".norm1", "gn", cin, cin, 0))
        L.append((p + ".conv1", "conv", cin, cout, 3))
        L.append((p + ".time_emb_proj", "linear", temb, cout, 0))
        L.append((p + ".norm2", "gn", cout, cout, 0))
        L.append((p + ".conv2", "conv", cout, cout, 3))
        if cin != cout:
            L.append((p + ".conv_shortcut", "conv", cin, cout, 1))

    def transformer(p, c, depth):
        # use_linear_projection: proj_in / proj_out are nn.Linear (SDXL), else 1x1 convolutions (SD1.5)
        kind, k = ("linear", 0) if cfg.use_linear_projection else ("conv", 1)
        L.append((p + ".norm", "gn", c, c, 0))
        L.append((p + ".proj_in", kind, c, c, k))
        for d in range(depth):
            t = p + f".transformer_blocks.{d}"
            L.append((t + ".norm1", "ln", c, c, 0))
            for n in ("to_q", "to_k", "to_v"):
                L.append((t + ".attn1." + n, "linear_nobias", c, c, 0))
            L.append((t + ".attn1.to_out.0", "linear", c, c, 0))
            L.append((t + ".norm2", "ln", c, c, 0))
            L.append((t + ".attn2.to_q", "linear_nobias", c, c, 0))
            L.append((t + ".attn2.to_k", "linear_nobias", cfg.cross_attention_dim, c, 0))
            L.append((t + ".attn2.to_v", "linear_nobias", cfg.cross_attention_dim, c, 0))
            L.append((t + ".attn2.to_out.0", "linear", c, c, 0))
            L.append((t + ".norm3", "ln", c, c, 0))
            L.append((t + ".ff.net.0.proj", "linear", c, 8 * c, 0))
            L.append((t + ".ff.net.2", "linear", 4 * c, c, 0))
        L.append((p + ".proj_out", kind, c, c, k))

    L.append(("conv_in", "conv", cfg.in_channels, ch[0], 3))
    L.append(("time_embedding.linear_1", "linear", ch[0], temb, 0))
    L.append(("time_embedding.linear_2", "linear", temb, temb, 0))
    if cfg.addition_embed:
        L.append(("add_embedding.linear_1", "linear", cfg.add_embed_in, temb, 0))
        L.append(("add_embedding.linear_2", "linear", temb, temb, 0))
    cin = ch[0]
    for i, cout in enumerate(ch):
        for j in range(cfg.layers_per_block):
            resnet(f"down_blocks.{i}.resnets.{j}", cin, cout)
            if cfg.down_attn[i]:
                transformer(f"down_blocks.{i}.attentions.{j}", cout, cfg.depth(i))
            cin = cout
        if i < len(ch) - 1:
            L.append((f"down_blocks.{i}.downsamplers.0.conv", "conv", cout, cout, 3))
    resnet("mid_block.resnets.0", ch[-1], ch[-1])
    transformer("mid_block.attentions.0", ch[-1], cfg.depth(len(ch) - 1))
    resnet("mid_block.resnets.1", ch[-1], ch[-1])
    rev = list(reversed(ch))
    prev = rev[0]
    for i, cout in enumerate(rev):
        skip_in = rev[min(i + 1, len(ch) - 1)]
        for j in range(cfg.layers_per_block + 1):
            skip = skip_in if j == cfg.layers_per_block else cout
            rin = prev if j == 0 else cout
            resnet(f"up_blocks.{i}.resnets.{j}", rin + skip, cout)
            if cfg.up_attn[i]:
                transformer(f"up_blocks.{i}.attentions.{j}", cout, cfg.depth(len(ch) - 1 - i))
        if i < len(ch) - 1:
            L.append((f"up_blocks.{i}.upsamplers.0.conv", "conv", cout, cout, 3))
        prev = cout
    L.append(("conv_norm_out", "gn", ch[0], ch[0], 0))
    L.append(("conv_out", "conv", ch[0], cfg.out_channels, 3))
    return L


def init_params(cfg: UNetConfig, seed: int = 0, lora_b_std: float = 0.02,
                dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights.  Base layers: nn.Conv2d/nn.Linear default init (kaiming-uniform
    a=sqrt(5) -> U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias); norms affine (1, 0).
    LoRA: A kaiming-uniform(a=sqrt(5)), B ~ N(0, lora_b_std) (peft default B = 0 makes LoRA
    invisible; pass lora_b_std=0 for the reference's step-0 initialisation)."""
    g = torch.Generator().manual_seed(seed)
    P = {}

    def uni(shape, bound):
        return (torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1) * bound

    for name, kind, cin, cout, k in layer_table(cfg):
        if kind in ("gn", "ln"):
            P[name + ".weight"] = torch.ones(cout)
            P[name + ".bias"] = torch.zeros(cout)
            continue
        if kind == "conv":
            fan_in = cin * k * k
            P[name + ".weight"] = uni((cout, cin, k, k), fan_in ** -0.5)
            P[name + ".bias"] = uni((cout,), fan_in ** -0.5)
        else:
            P[name + ".weight"] = uni((cout, cin), cin ** -0.5)
            if kind == "linear":
                P[name + ".bias"] = uni((cout,), cin ** -0.5)
        if _is_lora_target(name):
            r = cfg.lora_rank
            if kind == "conv":
                P[name + ".lora_A.weight"] = uni((r, cin, k, k), (cin * k * k) ** -0.5)
                P[name + ".lora_B.weight"] = torch.randn((cout, r, 1, 1), generator=g) * lora_b_std
            else:
                P[name + ".lora_A.weight"] = uni((r, cin), cin ** -0.5)
                P[name + ".lora_B.weight"] = torch.randn((cout, r), generator=g) * lora_b_std
    return {k: v.to(dtype) for k, v in P.items()}


def lora_keys(P):
    return [k for k in P if ".lora_" in k]


# ---------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------
def _round_grad(g):
    return g.to(torch.bfloat16).to(g.dtype)


def _q(x, on, grad=False):
    """bf16 rounding with a straight-through gradient; grad=True also rounds the gradient to bf16 (a hook:
    the forward is the same tensor either way)."""
    if not on:
        return x
    y = x + (x.to(torch.bfloat16).to(x.dtype) - x).detach()
    if grad and y.requires_grad:
        y.register_hook(_round_grad)
    return y


def _qg(x, on):
    """x itself, its gradient rounded to bf16 (a hook on x: only for a tensor that has this one use)."""
    if on and x.requires_grad:
        x.register_hook(_round_grad)
    return x


class UNetRef:
    """Functional UNet over a flat parameter dict.  use_lora=False gives the frozen teacher.

    round_grads (with emulate_bf16) rounds the gradients the CUDA backward (pcm_b200/unet.py) stores in
    bf16: those of every GEMM output but eps (conv_out's input gradient is computed from the fp32 d_eps),
    of every LoRA down-projection T, GroupNorm / LayerNorm output, attention output and GEGLU output, of
    a skip concatenation (add_bf16 then sums two bf16 gradients) and of an upsampler's nearest-neighbour
    output (upsample2x_bwd sums four bf16 gradients).  A time-embedding row vector takes its gradient
    before the rounding: the GroupNorm backward sums it over the pixels in fp32.  The softmax probabilities are
    left alone: the flash backward never stores dP, it rounds dS = P (dP - delta) in registers."""

    def __init__(self, cfg: UNetConfig, params: Dict[str, torch.Tensor], use_lora: bool = True,
                 emulate_bf16: bool = False, round_grads: bool = False):
        self.cfg, self.P, self.use_lora, self.emu = cfg, params, use_lora, emulate_bf16
        self.rg = emulate_bf16 and round_grads
        self.scale = cfg.lora_alpha / cfg.lora_rank
        self.taps = {}  # optional activation taps for layer-wise parity tests

    # -- primitives -------------------------------------------------------------------------
    def w(self, name):
        return _q(self.P[name], self.emu)

    def conv(self, name, x, stride=1, extra=None, rowvec=None):
        """Conv2d (+ peft LoRA branch) (+ fused additive terms), rounded once like the GEMM epilogue.
        rowvec: a per-sample [B, C, 1, 1] term (the time embedding); the GroupNorm backward sums its
        gradient in fp32 before it rounds the convolution's output gradient."""
        W = self.w(name + ".weight")
        k = W.shape[-1]
        y = F.conv2d(x, W, self.P.get(name + ".bias"), stride=stride, padding=k // 2)
        if self.use_lora and (name + ".lora_A.weight") in self.P:
            t = F.conv2d(x, self.w(name + ".lora_A.weight"), None, stride=stride, padding=k // 2)
            t = _q(t, self.emu, self.rg)
            y = y + F.conv2d(t, self.w(name + ".lora_B.weight") * self.scale)
        if extra is not None:
            y = y + extra
        if rowvec is not None:
            y = _qg(y, self.rg) + rowvec
            return _q(y, self.emu)
        return _q(y, self.emu, self.rg and name != "conv_out")

    def linear(self, name, x, extra=None, act=None):
        y = F.linear(x, self.w(name + ".weight"), self.P.get(name + ".bias"))
        if self.use_lora and (name + ".lora_A.weight") in self.P:
            t = _q(F.linear(x, self.w(name + ".lora_A.weight")), self.emu, self.rg)
            y = y + F.linear(t, self.w(name + ".lora_B.weight") * self.scale)
        if extra is not None:
            y = y + extra
        if act == "silu":
            y = F.silu(y)
        return _q(y, self.emu, self.rg)

    def gn(self, name, x, eps, silu):
        y = F.group_norm(x, self.cfg.norm_num_groups, self.P[name + ".weight"], self.P[name + ".bias"], eps)
        if silu:
            y = F.silu(y)
        return _q(y, self.emu, self.rg)

    def ln(self, name, x):
        return _q(F.layer_norm(x, (x.shape[-1],), self.P[name + ".weight"], self.P[name + ".bias"], 1e-5), self.emu,
                  self.rg)

    def attention(self, q, k, v, H=None):
        B, S, Cc = q.shape
        H = H or self.cfg.num_heads
        d = Cc // H
        q = q.view(B, S, H, d).transpose(1, 2)
        k = k.view(B, k.shape[1], H, d).transpose(1, 2)
        v = v.view(B, v.shape[1], H, d).transpose(1, 2)
        outs = []
        blk = 1024 if (S > 1024 and not torch.is_grad_enabled()) else S   # bound the S x S scratch
        for i in range(0, S, blk):
            s = (q[:, :, i:i + blk] @ k.transpose(-1, -2)) * (d ** -0.5)
            p = torch.softmax(s, dim=-1)
            p = _q(p, self.emu)  # the flash kernels feed bf16 probabilities to the PV product
            outs.append(p @ v)
        o = (outs[0] if len(outs) == 1 else torch.cat(outs, dim=2)).transpose(1, 2).reshape(B, S, Cc)
        return _q(o, self.emu, self.rg)

    # -- blocks -----------------------------------------------------------------------------
    def resnet(self, p, x, st):
        cin, cout = x.shape[1], self.P[p + ".conv1.weight"].shape[0]
        h = self.gn(p + ".norm1", x, 1e-5, True)
        tproj = self.linear(p + ".time_emb_proj", st)                       # [B, cout]
        h = self.conv(p + ".conv1", h, rowvec=tproj[:, :, None, None])
        h = self.gn(p + ".norm2", h, 1e-5, True)
        sc = self.conv(p + ".conv_shortcut", x) if cin != cout else x
        return self.conv(p + ".conv2", h, extra=sc)

    def transformer(self, p, x, ctx, level=0):
        """Transformer2DModel: GN -> proj_in -> depth x BasicTransformerBlock -> proj_out -> + residual.
        use_linear_projection (SDXL): proj_in / proj_out are nn.Linear applied to [B, HW, C] tokens;
        otherwise 1x1 convolutions on NCHW (SD1.5) - the same contraction."""
        B, Cc, Hh, Ww = x.shape
        H = self.cfg.heads(level)
        r = x
        h = self.gn(p + ".norm", x, 1e-6, False)
        if self.cfg.use_linear_projection:
            h = h.permute(0, 2, 3, 1).reshape(B, Hh * Ww, Cc)
            h = self.linear(p + ".proj_in", h)
        else:
            h = self.conv(p + ".proj_in", h)
            h = h.permute(0, 2, 3, 1).reshape(B, Hh * Ww, Cc)
        for d in range(self.cfg.depth(level)):
            t = p + f".transformer_blocks.{d}"
            n = self.ln(t + ".norm1", h)
            a = self.attention(self.linear(t + ".attn1.to_q", n), self.linear(t + ".attn1.to_k", n),
                               self.linear(t + ".attn1.to_v", n), H)
            h = self.linear(t + ".attn1.to_out.0", a, extra=h)
            n = self.ln(t + ".norm2", h)
            a = self.attention(self.linear(t + ".attn2.to_q", n), self.linear(t + ".attn2.to_k", ctx),
                               self.linear(t + ".attn2.to_v", ctx), H)
            h = self.linear(t + ".attn2.to_out.0", a, extra=h)
            n = self.ln(t + ".norm3", h)
            u = self.linear(t + ".ff.net.0.proj", n)
            a_, g_ = u.chunk(2, dim=-1)
            gg = _q(a_ * F.gelu(g_), self.emu, self.rg)                      # GEGLU, exact-erf GELU
            h = self.linear(t + ".ff.net.2", gg, extra=h)
        if self.cfg.use_linear_projection:
            h = self.linear(p + ".proj_out", h, extra=r.permute(0, 2, 3, 1).reshape(B, Hh * Ww, Cc))
            return h.reshape(B, Hh, Ww, Cc).permute(0, 3, 1, 2)
        h = h.reshape(B, Hh, Ww, Cc).permute(0, 3, 1, 2)
        return self.conv(p + ".proj_out", h, extra=r)

    def _sinusoid(self, values, dim):
        half = dim // 2
        dt = self.P["conv_in.weight"].dtype
        f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=dt, device=values.device) / half)
        e = values[:, None].to(dt) * f[None]
        return torch.cat([torch.cos(e), torch.sin(e)], dim=-1)               # flip_sin_to_cos, shift 0

    def time_embed(self, timesteps, added_cond_kwargs=None):
        c0 = self.cfg.block_out_channels[0]
        emb = _q(self._sinusoid(timesteps, c0), self.emu)
        h = self.linear("time_embedding.linear_1", emb, act="silu")
        if not self.cfg.addition_embed:
            # every consumer applies SiLU to temb first (ResnetBlock2D), so SiLU is folded in here
            return self.linear("time_embedding.linear_2", h, act="silu")
        # SDXL "text_time": emb = time_embedding(t) + add_embedding(cat[text_embeds, sinusoid(time_ids)])
        temb = self.linear("time_embedding.linear_2", h)
        text_embeds, time_ids = added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"]
        B = time_ids.shape[0]
        tid = self._sinusoid(time_ids.flatten(), self.cfg.addition_time_embed_dim).reshape(B, -1)
        add = _q(torch.cat([text_embeds.to(tid.dtype), tid], dim=-1), self.emu)
        a = self.linear("add_embedding.linear_1", add, act="silu")
        return self.linear("add_embedding.linear_2", a, extra=temb, act="silu")

    def __call__(self, sample, timesteps, encoder_hidden_states, added_cond_kwargs=None):
        """sample [B,4,H,W], timesteps [B] int64, encoder_hidden_states [B,77,D] -> eps [B,4,H,W]
        added_cond_kwargs (SDXL): {"text_embeds" [B, 1280], "time_ids" [B, 6]}"""
        cfg = self.cfg
        dt = self.P["conv_in.weight"].dtype
        x = _q(sample.to(dt), self.emu)
        ctx = _q(encoder_hidden_states.to(dt), self.emu)
        st = self.time_embed(timesteps, added_cond_kwargs)
        x = self.conv("conv_in", x)
        skips = [x]
        nb = len(cfg.block_out_channels)
        for i in range(nb):
            for j in range(cfg.layers_per_block):
                x = self.resnet(f"down_blocks.{i}.resnets.{j}", x, st)
                if cfg.down_attn[i]:
                    x = self.transformer(f"down_blocks.{i}.attentions.{j}", x, ctx, i)
                skips.append(x)
            if i < nb - 1:
                x = self.conv(f"down_blocks.{i}.downsamplers.0.conv", x, stride=2)
                skips.append(x)
        x = self.resnet("mid_block.resnets.0", x, st)
        x = self.transformer("mid_block.attentions.0", x, ctx, nb - 1)
        x = self.resnet("mid_block.resnets.1", x, st)
        self.taps["mid"] = x
        for i in range(nb):
            for j in range(cfg.layers_per_block + 1):
                x = _qg(torch.cat([x, skips.pop()], dim=1), self.rg)
                x = self.resnet(f"up_blocks.{i}.resnets.{j}", x, st)
                if cfg.up_attn[i]:
                    x = self.transformer(f"up_blocks.{i}.attentions.{j}", x, ctx, nb - 1 - i)
            if i < nb - 1:
                x = _qg(F.interpolate(x, scale_factor=2.0, mode="nearest"), self.rg)
                x = self.conv(f"up_blocks.{i}.upsamplers.0.conv", x)
        x = self.gn("conv_norm_out", x, 1e-5, True)
        return self.conv("conv_out", x)


def count_params(cfg):
    P = init_params(cfg, 0)
    base = sum(v.numel() for k, v in P.items() if ".lora_" not in k)
    lora = sum(v.numel() for k, v in P.items() if ".lora_" in k)
    return base, lora
