"""UNet / LoRA configuration of the hot path (SD1.5 `UNet2DConditionModel` as constructed at
train_pcm_lora_sd15.py:840-852 and wrapped by peft at :866-885)."""
from dataclasses import dataclass
from typing import Tuple

# peft target-module suffixes, train_pcm_lora_sd15.py:868-883
LORA_TARGETS = ("to_q", "to_k", "to_v", "to_out.0", "proj_in", "proj_out", "ff.net.0.proj",
                "ff.net.2", "conv1", "conv2", "conv_shortcut", "downsamplers.0.conv",
                "upsamplers.0.conv", "time_emb_proj")


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    cross_attention_dim: int = 768
    num_heads: int = 8  # SD1.5's `attention_head_dim=8` is a head COUNT in diffusers 0.26.3
    norm_num_groups: int = 32
    down_attn: Tuple[bool, ...] = (True, True, True, False)
    lora_rank: int = 64
    lora_alpha: float = 8.0  # peft LoraConfig default -> scaling = 8 / r
    # SDXL-style extensions (train_pcm_lora_sdxl_adv.py; diffusers UNet2DConditionModel config of
    # stabilityai/stable-diffusion-xl-base-1.0): transformer blocks per attention level, heads per level,
    # Linear proj_in / proj_out, and the "text_time" additional embedding (added_cond_kwargs)
    transformer_layers_per_block: Tuple[int, ...] = ()      # () -> 1 everywhere
    heads_per_block: Tuple[int, ...] = ()                   # () -> num_heads everywhere
    use_linear_projection: bool = False
    addition_embed: bool = False                            # addition_embed_type == "text_time"
    addition_time_embed_dim: int = 256
    text_embed_dim: int = 1280                              # pooled text embedding width
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

    @property
    def lora_scale(self):
        return self.lora_alpha / self.lora_rank


LORA_RANKS = "8 <= r <= 256 with r % 8 == 0"


def check_lora_rank(r):
    """Raise ValueError unless r is a supported LoRA rank: 8 <= r <= 256, r % 8 == 0 (a [M, r] bf16 row of
    the rank-side operands must be a multiple of 16 bytes for TMA)."""
    if isinstance(r, bool) or not isinstance(r, int) or not (8 <= r <= 256 and r % 8 == 0):
        raise ValueError(f"unsupported LoRA rank {r!r}: the supported ranks are {LORA_RANKS}")
    return r


SD15 = UNetConfig()
# small configuration for fast parity tests (same topology, narrower)
TINY = UNetConfig(block_out_channels=(64, 128, 128, 128), cross_attention_dim=64, num_heads=2)
# SDXL base UNet (train_pcm_lora_sdxl_adv.py: 3 levels, DownBlock2D + 2 x CrossAttnDownBlock2D, transformer
# depth 1 / 2 / 10, 64-wide heads, 2048-d context, Linear projections, text_time embedding)
SDXL = UNetConfig(block_out_channels=(320, 640, 1280), down_attn=(False, True, True),
                  transformer_layers_per_block=(1, 2, 10), heads_per_block=(5, 10, 20),
                  cross_attention_dim=2048, use_linear_projection=True, addition_embed=True)
# narrow SDXL-shaped configuration for parity tests
TINY_XL = UNetConfig(block_out_channels=(64, 128, 128), down_attn=(False, True, True),
                     transformer_layers_per_block=(1, 2, 3), heads_per_block=(1, 2, 2),
                     cross_attention_dim=128, use_linear_projection=True, addition_embed=True,
                     addition_time_embed_dim=64, text_embed_dim=128)


def is_lora_target(name: str) -> bool:
    return any(name == t or name.endswith("." + t) for t in LORA_TARGETS)


def layer_table(cfg: UNetConfig):
    """Ordered (name, kind, cin, cout, ksize) for every parameterised layer, execution order.
    kind in {conv, linear, linear_nobias, gn, ln}."""
    L = []
    ch = cfg.block_out_channels
    temb = cfg.time_embed_dim

    def resnet(p, cin, cout):
        L.extend([(p + ".norm1", "gn", cin, cin, 0), (p + ".conv1", "conv", cin, cout, 3),
                  (p + ".time_emb_proj", "linear", temb, cout, 0), (p + ".norm2", "gn", cout, cout, 0),
                  (p + ".conv2", "conv", cout, cout, 3)])
        if cin != cout:
            L.append((p + ".conv_shortcut", "conv", cin, cout, 1))

    def transformer(p, c, depth):
        proj = ("linear", 0) if cfg.use_linear_projection else ("conv", 1)
        L.extend([(p + ".norm", "gn", c, c, 0), (p + ".proj_in", proj[0], c, c, proj[1])])
        for d in range(depth):
            t = p + f".transformer_blocks.{d}"
            L.extend([(t + ".norm1", "ln", c, c, 0),
                      (t + ".attn1.to_q", "linear_nobias", c, c, 0), (t + ".attn1.to_k", "linear_nobias", c, c, 0),
                      (t + ".attn1.to_v", "linear_nobias", c, c, 0), (t + ".attn1.to_out.0", "linear", c, c, 0),
                      (t + ".norm2", "ln", c, c, 0),
                      (t + ".attn2.to_q", "linear_nobias", c, c, 0),
                      (t + ".attn2.to_k", "linear_nobias", cfg.cross_attention_dim, c, 0),
                      (t + ".attn2.to_v", "linear_nobias", cfg.cross_attention_dim, c, 0),
                      (t + ".attn2.to_out.0", "linear", c, c, 0),
                      (t + ".norm3", "ln", c, c, 0),
                      (t + ".ff.net.0.proj", "linear", c, 8 * c, 0), (t + ".ff.net.2", "linear", 4 * c, c, 0)])
        L.append((p + ".proj_out", proj[0], c, c, proj[1]))

    L.append(("conv_in", "conv", cfg.in_channels, ch[0], 3))
    L.append(("time_embedding.linear_1", "linear", ch[0], temb, 0))
    L.append(("time_embedding.linear_2", "linear", temb, temb, 0))
    if cfg.addition_embed:   # TimestepEmbedding(projection_class_embeddings_input_dim, time_embed_dim)
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
