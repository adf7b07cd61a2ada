"""The VAE's host code (pcm_b200/vae.py) on CPU: the oracle's parameter inventory, the loader in both attention
spellings, the asymmetric stride-2 downsample plan, the encoder and decoder with every kernel interpreted
against the oracle (oracle/vae_ref.py), and the wide-image GEMM descriptors the host builds against
pcm_gemm_check."""
import ctypes
import json
import os

import pytest
import torch
import torch.nn.functional as F

import vae_interp
from gemm_interp import interp_gemm
from oracle import vae_ref
from pcm_b200 import ops, vae

BF16 = torch.bfloat16


def test_inventory_sd15():
    """The SD1.5 VAE: 83,653,863 parameters, 34,163,664 in the encoder with quant_conv, 49,490,199 in the
    decoder with post_quant_conv; the product's layer table holds the same tensors."""
    enc, dec = vae_ref.count_params(vae_ref.SD15)
    assert (enc, dec, enc + dec) == (34_163_664, 49_490_199, 83_653_863)
    cfg = vae.VAEConfig()
    assert vae.layer_table(cfg) == vae_ref.layer_table(vae_ref.SD15)
    sd = vae.synthetic_state_dict(cfg)
    assert sum(v.numel() for v in sd.values()) == 83_653_863


def _write(tmp, sd, cfg, legacy):
    from safetensors.torch import save_file
    d = os.path.join(tmp, "vae")
    os.makedirs(d, exist_ok=True)
    out = {}
    for k, v in sd.items():
        if legacy and ".attentions.0." in k:
            for new, old in (("to_q", "query"), ("to_k", "key"), ("to_v", "value"), ("to_out.0", "proj_attn")):
                k = k.replace(f".attentions.0.{new}.", f".attentions.0.{old}.")
        out[k] = v.contiguous()
    save_file(out, os.path.join(d, "diffusion_pytorch_model.safetensors"))
    conf = {"_class_name": "AutoencoderKL", "in_channels": 3, "out_channels": 3, "latent_channels": 4,
            "block_out_channels": list(cfg.block_out_channels), "layers_per_block": cfg.layers_per_block,
            "norm_num_groups": cfg.norm_num_groups, "scaling_factor": cfg.scaling_factor, "sample_size": 512}
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(conf, f)


@pytest.mark.parametrize("legacy", [False, True])
def test_loader_both_spellings(tmp_path, legacy):
    cfg = vae.VAEConfig(block_out_channels=(64, 128), layers_per_block=1, scaling_factor=0.13025)
    sd = vae.synthetic_state_dict(cfg, seed=5)
    _write(str(tmp_path), sd, cfg, legacy)
    v = vae.AutoencoderKL.from_pretrained(str(tmp_path), subfolder="vae", device="cpu")
    assert v.config.scaling_factor == 0.13025 and v.cfg.block_out_channels == (64, 128)
    ref = vae.AutoencoderKL(cfg, sd, "cpu")
    for p in ("encoder.mid_block.attentions.0", "decoder.mid_block.attentions.0"):
        assert torch.equal(v.layers[p].w_qkv, ref.layers[p].w_qkv)
        assert torch.equal(v.layers[p].w_out, ref.layers[p].w_out)
        assert torch.equal(v.layers[p].b_qkv, ref.layers[p].b_qkv)
        qkv = torch.cat([sd[f"{p}.{n}.weight"] for n in ("to_q", "to_k", "to_v")]).to(BF16)
        assert torch.equal(ops.kblock(qkv), v.layers[p].w_qkv)
    assert torch.equal(v.layers["encoder.conv_in"].w_c4[..., 3], torch.zeros(64, 3, 3, dtype=BF16))


def test_loader_rejects_mismatched_config(tmp_path):
    cfg = vae.VAEConfig(block_out_channels=(64, 128), layers_per_block=1)
    _write(str(tmp_path), vae.synthetic_state_dict(cfg), vae.VAEConfig(block_out_channels=(64, 192),
                                                                        layers_per_block=1), False)
    with pytest.raises((ValueError, KeyError)):
        vae.AutoencoderKL.from_pretrained(str(tmp_path), device="cpu")


@pytest.mark.parametrize("W", [32, 256])
def test_downsample_plan(monkeypatch, W):
    """Downsample2D(padding=0): the parity-plane K program with the (0, 0), (1, 0), (0, +1) tap table is
    F.conv2d(F.pad(x, (0, 1, 0, 1)), stride=2)."""
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    cfg = vae.VAEConfig(block_out_channels=(64, 128), layers_per_block=1)
    v = vae.AutoencoderKL(cfg, vae.synthetic_state_dict(cfg, seed=1), "cpu")
    g = torch.Generator().manual_seed(0)
    H = 6
    x = torch.randn(2, H, W, 64, generator=g).to(BF16)
    out = v.conv("encoder.down_blocks.0.downsamplers.0.conv", x, stride=2)
    sd = vae.synthetic_state_dict(cfg, seed=1)
    w = sd["encoder.down_blocks.0.downsamplers.0.conv.weight"].to(BF16).float()
    b = sd["encoder.down_blocks.0.downsamplers.0.conv.bias"]
    ref = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), w, b, stride=2).permute(0, 2, 3, 1)
    assert out.shape == (2, H // 2, W // 2, 64)
    torch.testing.assert_close(out.float(), ref.to(BF16).float(), rtol=1e-2, atol=1e-2)
    assert (out.float() - ref).abs().max() <= 2 ** -7 * ref.abs().max()


def _bound(cuda, emu, f64):
    """(max |host - bf16 oracle|, max |bf16 oracle - float64 network|): two bf16 implementations that round at
    the same points but sum in different orders flip single bf16 roundings, which then propagate like any
    other bf16 rounding; each is within the oracle's own distance to the exact network, so they are within
    twice that distance of each other."""
    err = (cuda.double() - emu.double()).abs().max().item()
    own = (emu.double() - f64).abs().max().item()
    return err, own


def test_vae_host_vs_oracle(monkeypatch):
    vae_interp.install(monkeypatch)
    cfg_o = vae_ref.TINY
    cfg = vae.VAEConfig(block_out_channels=cfg_o.block_out_channels, layers_per_block=cfg_o.layers_per_block)
    P = vae_ref.init_params(cfg_o, seed=2)
    v = vae.AutoencoderKL(cfg, P, "cpu")
    g = torch.Generator().manual_seed(1)
    images = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1
    emu = vae_ref.VAERef(cfg_o, P, emulate_bf16=True)
    exact = vae_ref.VAERef(cfg_o, {k: t.double() for k, t in P.items()})
    dist = v.encode(images).latent_dist
    mean_e, logvar_e = emu.encode(images)
    mean_x, _ = exact.encode(images.double())
    err, own = _bound(dist.mean, mean_e, mean_x)
    assert err <= 2 * own, (err, own)
    torch.testing.assert_close(dist.logvar, logvar_e, rtol=0, atol=2 * own)
    assert torch.equal(dist.std, torch.exp(0.5 * dist.logvar))
    assert torch.equal(dist.mode(), dist.mean)
    z = dist.sample(torch.Generator().manual_seed(3))
    n = torch.randn(dist.mean.shape, generator=torch.Generator().manual_seed(3))
    assert torch.equal(z, dist.mean + dist.std * n)
    lat = torch.randn(2, 4, 16, 16, generator=g)
    img = v.decode(lat).sample
    ref_e = emu.decode(lat)
    ref_x = exact.decode(lat.double())
    err, own = _bound(img, ref_e, ref_x)
    assert img.shape == (2, 3, 32, 32)
    assert err <= 2 * own, (err, own)
    # the pipeline's decode + postprocess
    out = torch.empty(2, 3, 32, 32)
    u8 = torch.empty(2, 32, 32, 3, dtype=torch.uint8)
    v.decode_images((lat * 0.18215).permute(0, 2, 3, 1).contiguous(), 0.18215, out, u8)
    ref = (v.decode(lat * 0.18215 / 0.18215).sample / 2 + 0.5).clamp(0, 1)
    torch.testing.assert_close(out, ref, rtol=0, atol=1e-6)
    assert torch.equal(u8, (out.permute(0, 2, 3, 1) * 255).round().to(torch.uint8))


def test_wide_descriptors_pass_check(monkeypatch):
    """The descriptors the host builds for 3x3 and stride-2 convolutions of images 256, 512 and 1024 pixels
    wide (TMA boxes of 128 pixels of one row) pass pcm_gemm_check."""
    from pcm_b200 import _lib
    lib = _lib.lib()
    seen = []

    class Checker:
        def pcm_gemm(self, d, stream):
            seen.append((d._obj.geoW, lib.pcm_gemm_plan_rows(d)))
            return lib.pcm_gemm_check(d)

        def pcm_last_error(self):
            return lib.pcm_last_error()

    monkeypatch.setattr(_lib, "lib", lambda: Checker())
    monkeypatch.setattr(ops, "_stream", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(ops, "_NUM_SMS", 132)
    cfg = vae.VAEConfig(block_out_channels=(128, 256), layers_per_block=1)
    v = vae.AutoencoderKL(cfg, vae.synthetic_state_dict(cfg), "cpu")
    for W in (256, 512, 1024):
        x = torch.zeros(1, 4, W, 128, dtype=BF16)
        v.conv("encoder.down_blocks.0.resnets.0.conv1", x)
        v.conv("encoder.down_blocks.0.downsamplers.0.conv", x, stride=2)
        x = torch.zeros(1, 4, W, 256, dtype=BF16)
        v.conv("encoder.down_blocks.1.resnets.0.conv2", x, residual=torch.zeros(1, 4, W, 256, dtype=BF16))
    assert sorted({w for w, _ in seen}) == [128, 256, 512, 1024]
