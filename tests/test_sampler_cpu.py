"""HOST logic of the few-step sampler (pcm_b200/sampling.py) on CPU: the timestep / coefficient schedule
against the reference's own scheduler code (tests/golden/sampler_math.pt), the pcm_lora_fuse table, the
sampling loop with every kernel interpreted (tests/sampler_interp.py) against the CPU oracle
(tests/sample_oracle.py), argument errors, adapter round trip and the trainer's validation flags."""
import dataclasses
import math
import os

import pytest
import torch

import sampler_interp
from gemm_interp import BF16, build_net
from sample_oracle import sample_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sampler_math.pt")


def _sampler(net, **kw):
    from pcm_b200.sampling import PCMSampler
    return PCMSampler(net, **kw)


def test_timesteps_and_coefficients_match_the_reference_scheduler():
    from pcm_b200 import sampling
    gold = torch.load(GOLDEN)
    acp = gold["alphas_cumprod"]
    for n in gold["ns"]:
        d = gold[f"n{n}"]
        ts = sampling.trailing_timesteps(n)
        assert ts.tolist() == d["timesteps"].tolist()
        assert sampling.previous_timesteps(ts, n).tolist() == d["prev_timesteps"].tolist()
        coef = sampling.step_coefficients(acp, n)
        for i, (t, sa, ss, sap, ssp) in enumerate(coef):
            a, ap = float(d["alpha_t"][i]), float(d["alpha_prev"][i])
            assert (sa, ss, sap, ssp) == (math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap))
        # one DDIM update of the fixture (predicted_origin + ddim_step formula of the reference) through the
        # interpreted step kernel's arithmetic
        i = d["step_i"]
        _, sa, ss, sap, ssp = coef[i]
        x, e = d["x"].double(), d["eps"].double()
        x0 = (x - ss * e) / sa
        ours = (sap * x0 + ssp * e)
        assert torch.allclose(ours, d["x_prev"].double(), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("rank", [8, 64, 136, 256])
def test_fuse_table_writes_every_lora_operand_element_once(monkeypatch, rank):
    from pcm_b200 import config
    cfg = dataclasses.replace(config.TINY_XL, lora_rank=rank)
    net, _ = build_net(cfg)
    inf, table, work = net.fused_inference_net()
    rows = sampler_interp.fuse_rows(table.data_ptr(), table.shape[0])
    assert len(rows) == len(net.lora_layers)
    assert sorted(r["a_off"] for r in rows) == sorted(L.lora.a_off for L in net.lora_layers)
    base = inf.fused_weights.data_ptr()
    count = torch.zeros(inf.fused_weights.numel(), dtype=torch.int32)
    for r in rows:
        assert r["r"] == rank and r["K"] % 64 == 0 and r["n"] % 64 == 0
        v = count[(r["dst"] - base) // 2:][:r["K"] * r["ntot"]].view(r["K"] // 64, r["ntot"], 64)
        v[:, r["n0"]:r["n0"] + r["n"]] += 1
    assert torch.equal(count, torch.ones_like(count))
    assert work == sum((r["n"] // 64) * (r["K"] // 64) for r in rows)
    # the interpreted kernel writes every element (NaN sentinels) and leaves the sources alone
    sampler_interp.install(monkeypatch)
    inf.fused_weights.fill_(float("nan"))
    srcs = [t.clone() for t in (net.temb_group.w_stack, *[ch.w_stack for ch in net.ctx_group.chunks])]
    from pcm_b200 import ops
    ops.lora_fuse(net.lora_master, table, work, net.scale)
    assert not inf.fused_weights.float().isnan().any()
    assert all(torch.equal(a, b) for a, b in zip(srcs, (net.temb_group.w_stack,
                                                       *[ch.w_stack for ch in net.ctx_group.chunks])))
    # every fused operand is W + s B A of its layers (one Linear, one conv, one stack member)
    from gemm_interp import b_matrix
    from pcm_b200 import ops as O
    for name in ("down_blocks.1.attentions.0.proj_in", "down_blocks.0.resnets.0.conv1"):
        L, L2 = net.layers[name], inf.layers[name]
        taps = L.k * L.k if L.kind == "conv" else 1
        A = net.lora_master[L.lora.a_off:L.lora.a_off + rank * taps * L.cin].view(rank, -1)
        Bm = net.lora_master[L.lora.b_off:L.lora.b_off + L.cout * rank].view(L.cout, rank)
        want = (b_matrix(O.bsrc(L.w_fwd)).float() + net.scale * (Bm.double() @ A.double()).float()).to(BF16)
        assert torch.equal(b_matrix(O.bsrc(L2.w_fwd)), want)


def _inputs(ocfg, P, hw, seed=5):
    g = torch.Generator().manual_seed(seed)
    pe = torch.randn(P, 77, ocfg.cross_attention_dim, generator=g)
    ne = torch.randn(P, 77, ocfg.cross_attention_dim, generator=g)
    kw = {}
    if getattr(ocfg, "addition_embed", False):
        kw = dict(text_embeds=torch.randn(P, ocfg.text_embed_dim, generator=g),
                  negative_text_embeds=torch.zeros(P, ocfg.text_embed_dim),
                  time_ids=torch.tensor([hw * 8, hw * 8, 0, 0, hw * 8, hw * 8]))
    return pe, ne, kw


@pytest.mark.parametrize("cfg_name", ["TINY", "TINY_XL"])
@pytest.mark.parametrize("n", [1, 2, 4])
@pytest.mark.parametrize("guidance", [1.0, 7.5])
def test_sampler_host_sequence_matches_the_oracle(monkeypatch, cfg_name, n, guidance):
    from oracle import unet_ref
    from pcm_b200 import config
    ocfg = getattr(unet_ref, cfg_name)
    Pw = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    net, _ = build_net(getattr(config, cfg_name), sd=Pw)
    sampler_interp.install(monkeypatch)
    sampler = _sampler(net)
    P, nipp, hw = 1, 2, 8
    pe, ne, kw = _inputs(ocfg, P, hw)
    lat = torch.randn(P * nipp, 4, hw, hw, generator=torch.Generator().manual_seed(9))
    out = sampler(pe, ne, num_inference_steps=n, guidance_scale=guidance, num_images_per_prompt=nipp,
                  height=8 * hw, width=8 * hw, latents=lat, **kw)
    assert out.shape == (P * nipp, 4, hw, hw) and out.dtype == torch.float32
    rep = lambda t: t.repeat_interleave(nipp, 0)  # noqa: E731
    addc = nadd = None
    if kw:
        tid = kw["time_ids"].reshape(1, -1).expand(P * nipp, -1)
        addc = dict(text_embeds=rep(kw["text_embeds"]), time_ids=tid)
        nadd = dict(text_embeds=rep(kw["negative_text_embeds"]), time_ids=tid)
    ref = sample_ref(ocfg, Pw, rep(pe), rep(ne), num_inference_steps=n, latents=lat, guidance_scale=guidance,
                     added_cond=addc, negative_added_cond=nadd, emulate_bf16=True)
    rel = ((out.double() - ref.double()).norm() / ref.double().norm()).item()
    # bf16 network evaluations against the oracle's emulation (same kind of bound as test_unet_host_cpu.py);
    # guidance 7.5 amplifies the eps difference of the two halves
    assert rel < (2e-2 if guidance <= 1 else 5e-2), rel


def test_argument_errors(monkeypatch):
    from pcm_b200 import config
    net, _ = build_net(config.TINY)
    sampler_interp.install(monkeypatch)
    s = _sampler(net)
    pe = torch.randn(2, 77, 64)
    ok = dict(num_inference_steps=2, height=64, width=64)
    for bad in (dict(ok, num_inference_steps=0), dict(ok, num_inference_steps=1001)):
        with pytest.raises(ValueError):
            s(pe, **bad)
    with pytest.raises(ValueError):
        s(torch.randn(2, 77, 32), **ok)                          # wrong embedding width
    with pytest.raises(ValueError):
        s(pe, torch.randn(1, 77, 64), guidance_scale=7.5, **ok)  # batch mismatch
    with pytest.raises(ValueError):
        s(pe, guidance_scale=7.5, **ok)                          # no negative embedding
    with pytest.raises(ValueError):
        s(pe, latents=torch.randn(1, 4, 8, 8), **ok)             # latents of another batch
    with pytest.raises(ValueError):
        s(pe, **dict(ok, height=60))
    with pytest.raises(ValueError):
        _sampler(net, prediction_type="sample")
    xl, _ = build_net(config.TINY_XL)
    sx = _sampler(xl)
    pe = torch.randn(1, 77, 128)
    with pytest.raises(ValueError):
        sx(pe, **ok)                                             # missing SDXL conditions
    with pytest.raises(ValueError):
        sx(pe, pe, guidance_scale=7.5, text_embeds=torch.randn(1, 128), time_ids=torch.zeros(6), **ok)


def test_adapter_round_trip(tmp_path, monkeypatch):
    import types
    from pcm_b200 import config
    from pcm_b200.sampling import load_lora_adapter
    from pcm_b200.train_pcm_lora_sd15 import save_lora
    net, sd = build_net(config.TINY)
    sampler_interp.install(monkeypatch)
    a = _sampler(net)
    save_lora(types.SimpleNamespace(unet=net), config.TINY, str(tmp_path))
    ad = load_lora_adapter(str(tmp_path))
    assert set(ad) == set(net.lora_state_dict())
    base = {k: v for k, v in sd.items() if ".lora_" not in k}
    net2, _ = build_net(config.TINY, sd={**base, **ad})
    b = _sampler(net2)
    assert torch.equal(a.net.fused_weights, b.net.fused_weights)


def test_validation_flags():
    from pcm_b200 import train_pcm_lora_sd15 as T
    a = T.parse_args(["--synthetic", "--validation_prompt_embeds", "v.pt"])
    assert a.validation_prompt_embeds == "v.pt"
    b = T.parse_args(["--synthetic"])
    assert b.validation_prompt_embeds is None and not T.validation_enabled(b)
    assert T.validation_enabled(a)
    assert T.validation_guidances(config_sdxl=False) == (1.0, 7.5)
    assert T.validation_guidances(config_sdxl=True) == (1.0,)
