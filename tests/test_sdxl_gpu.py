"""SDXL-shaped UNet on the CUDA path (SURVEY section 8f-2, BASELINE config 4 without the adversarial
term): three levels (DownBlock2D, 2 x CrossAttnDownBlock2D), transformer depth > 1, 64-wide heads,
Linear proj_in / proj_out, `added_cond_kwargs` (text_time embedding), zero unconditional embeddings,
40 DDIM steps - train_pcm_lora_sdxl_adv.py:307-366, 1094-1133, 1215-1221.  Parity against the oracle
(oracle/unet_ref.py, SDXL options restated from the diffusers config) on a narrow configuration."""
import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _setup(B, hw, seed=0):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    P = unet_ref.init_params(unet_ref.TINY_XL, seed)
    batch = pcm_ref.make_batch(unet_ref.TINY_XL, B, hw, seed=seed, num_ddim=40, zero_uncond=True)
    return unet_ref.TINY_XL, config.TINY_XL, P, batch


def test_sdxl_unet_forward_backward(cuda):
    from oracle import unet_ref
    from pcm_b200.unet import UNetB200
    B, hw = 2, 16
    ocfg, pcfg, P, batch = _setup(B, hw)
    x, ctx = batch["latents"], batch["prompt_embeds"]
    ts = torch.tensor([999, 24])
    addc = dict(text_embeds=batch["text_embeds"], time_ids=batch["time_ids"])
    net = UNetB200(pcfg, P, cuda)
    dev_add = (batch["text_embeds"].to(cuda).to(BF), batch["time_ids"].to(cuda))
    dctx = ctx.to(cuda).to(BF).reshape(B * 77, -1)
    outs = {}
    for lora in (True, False):
        ref = unet_ref.UNetRef(ocfg, P, use_lora=lora, emulate_bf16=True)(x, ts, ctx, addc)
        out = _nchw(net.forward(_nhwc(x).to(cuda), ts.to(cuda), dctx, lora=lora, added_cond=dev_add)).cpu()
        err = (out - ref).abs()
        assert err.max().item() <= 3e-2 * ref.abs().max().item(), (lora, err.max().item())
        assert err.mean().item() <= 1e-2 * ref.pow(2).mean().sqrt().item(), (lora, err.mean().item())
        outs[lora] = out
    assert (outs[True] - outs[False]).abs().max().item() > 1e-3
    # the added conditions matter
    other = (torch.zeros_like(dev_add[0]), dev_add[1])
    out2 = _nchw(net.forward(_nhwc(x).to(cuda), ts.to(cuda), dctx, lora=True, added_cond=other)).cpu()
    assert (out2 - outs[True]).abs().max().item() > 1e-3
    with pytest.raises(ValueError):
        net.forward(_nhwc(x).to(cuda), ts.to(cuda), dctx, lora=True)
    # backward with a fixed cotangent
    G = torch.randn(B, 4, hw, hw, generator=torch.Generator().manual_seed(7)) / (B * 4 * hw * hw)
    Pg = {k: (v.clone().requires_grad_(True) if ".lora_" in k else v) for k, v in P.items()}
    eps = unet_ref.UNetRef(ocfg, Pg, use_lora=True, emulate_bf16=True)(x, ts, ctx, addc)
    (eps * G).sum().backward()
    ref_g = {k: v.grad for k, v in Pg.items() if ".lora_" in k}
    net.forward(_nhwc(x).to(cuda), ts.to(cuda), dctx, lora=True, save=True, added_cond=dev_add)
    net.backward(_nhwc(G).to(cuda))
    torch.cuda.synchronize()
    g = net.lora_grad_dict()
    num = sum((g[k].cpu().float() - rg).pow(2).sum().item() for k, rg in ref_g.items())
    den = sum(rg.pow(2).sum().item() for rg in ref_g.values())
    dot = sum((g[k].cpu().float() * rg).sum().item() for k, rg in ref_g.items())
    n1 = sum(g[k].float().pow(2).sum().item() for k in ref_g)
    assert (num / den) ** 0.5 <= 5e-2 and dot / (n1 ** 0.5 * den ** 0.5) >= 0.998


def test_sdxl_step_loss(cuda):
    """Whole PCM step on the SDXL-shaped network: 40 DDIM steps, zero unconditional embeddings, added
    conditions on all four passes; merged batch-3B pass; loss vs the oracle at N = 4 * 4 * 32 * 32."""
    from oracle import pcm_ref
    from pcm_b200.step import PCMTrainStep
    B, hw, mp = 4, 32, 4
    ocfg, pcfg, P, batch = _setup(B, hw, seed=1)
    ref = pcm_ref.pcm_step_ref(ocfg, P, batch, multiphase=mp, num_ddim=40, emulate_bf16=True, need_grad=False)
    st = PCMTrainStep(pcfg, P, cuda, batch=B, height=hw, width=hw, multiphase=mp, num_ddim_timesteps=40,
                      keep_debug=True)
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF), batch["uncond_prompt_embeds"].to(BF),
                   text_embeds=batch["text_embeds"].to(BF), time_ids=batch["time_ids"])
    st.forward_backward()
    torch.cuda.synchronize()
    assert torch.equal(st.start_t.cpu(), ref["start_timesteps"]) and torch.equal(st.t.cpu(), ref["timesteps"])
    assert torch.equal(st.end_t.cpu(), ref["end_timesteps"])
    rel = lambda a, b: ((a.float() - b.float()).norm() / b.float().norm()).item()
    assert rel(_nchw(st.x_prev).cpu(), ref["x_prev"]) < 2e-2
    assert rel(_nchw(st.model_pred).cpu(), ref["model_pred"]) < 2e-2
    loss, rloss = st.loss.item(), ref["loss"].item()
    print(f"[sdxl tiny] loss {loss:.6f} oracle {rloss:.6f} rel {abs(loss - rloss) / rloss:.2e}")
    assert abs(loss - rloss) <= 2e-2 * abs(rloss), (loss, rloss)
    st.optimizer_step()
    torch.cuda.synchronize()
    assert st.unet.lora_grad.abs().max().item() == 0.0
    with pytest.raises(ValueError):
        st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                       batch["prompt_embeds"].to(BF), batch["uncond_prompt_embeds"].to(BF))
