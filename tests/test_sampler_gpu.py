"""The few-step sampler on the GPU: pcm_lora_fuse against float64 torch on every kind of operand a LoRA
target's frozen weight lives in, pcm_sample_step against float64, the fused forward against the trained
network's unfused LoRA forward at SD1.5 width, the whole sampler against the CPU oracle (eager == graph
replay, bit for bit), non-interference with a captured training step, and the trainer's validation."""
import dataclasses
import gc

import pytest
import torch

from sample_oracle import sample_ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _unblock(w):
    """K-blocked [K/64, N, 64] -> [N, K]."""
    return w.permute(1, 0, 2).reshape(w.shape[1], -1)


@pytest.mark.parametrize("rank", [8, 64, 136, 256])
def test_lora_fuse_matches_float64(cuda, rank):
    from pcm_b200 import config, ops, weights
    from pcm_b200.unet import UNetB200
    cfg = dataclasses.replace(config.TINY_XL, lora_rank=rank)
    sd = weights.synthetic_state_dict(cfg, 1, lora_b_std=0.5)
    net = UNetB200(cfg, sd, cuda, need_backward=False)
    inf, table, work = net.fused_inference_net()
    before = [t.clone() for t in (net.temb_group.w_stack, net.ctx_group.chunks[0].w_stack)]
    ops.lora_fuse(net.lora_master, table, work, net.scale)
    first = inf.fused_weights.clone()
    ops.lora_fuse(net.lora_master, table, work, net.scale)
    torch.cuda.synchronize()
    assert torch.equal(first, inf.fused_weights)          # repeats are bitwise equal
    assert all(torch.equal(a, b) for a, b in zip(before, (net.temb_group.w_stack, net.ctx_group.chunks[0].w_stack)))
    s = net.scale

    def want(name):
        """(float64 W + s B A, the magnitude |W| + s |B| |A|) of one layer, [n, K] in the OHWI K order"""
        W = sd[name + ".weight"]
        W = (W.permute(0, 2, 3, 1) if W.dim() == 4 else W).reshape(W.shape[0], -1).to(BF).double()
        A = sd[name + ".lora_A.weight"]
        A = (A.permute(0, 2, 3, 1) if A.dim() == 4 else A).reshape(rank, -1).double()
        Bm = sd[name + ".lora_B.weight"].reshape(-1, rank).double()
        return W + s * (Bm @ A), W.abs() + s * (Bm.abs() @ A.abs())

    def stacked(names):
        parts = [want(n) for n in names]
        return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])

    def check(got, exp, mag):
        """got within 1 bf16 ulp of the float64 result, beyond the error bound of an fp32 rank sum
        ((r + 2) 2^-24 of the magnitudes |W| + s |B| |A|, which only matters where W and s B A cancel), and
        equal to the float64 result rounded to bf16 for all but 1 % of the elements."""
        got = got.double().cpu()
        assert got.shape == exp.shape
        _, e2 = torch.frexp(exp)
        ulp = torch.ldexp(torch.ones_like(exp), e2 - 8)                           # bf16: 8 significant bits
        bound = ulp + (rank + 2) * 2.0 ** -24 * mag
        err = (got - exp).abs()
        i = int((err - bound).argmax())
        assert (err <= bound).all(), (exp.flatten()[i].item(), got.flatten()[i].item(), ulp.flatten()[i].item())
        assert (got != exp.to(BF).double()).double().mean().item() < 0.01        # < 1 % off the nearest

    lin = "down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_out.0"
    check(_unblock(inf.layers[lin].w_fwd), *want(lin))
    conv = "down_blocks.1.resnets.0.conv1"
    check(_unblock(inf.layers[conv].w_fwd), *want(conv))
    lead = "down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q"
    check(_unblock(inf.groups[lead].w_stack), *stacked([lead[:-1] + c for c in "qkv"]))
    check(_unblock(inf.temb_group.w_stack), *stacked(inf.temb_group.names))
    ch = inf.ctx_group.chunks[0]
    names = [n for G in net.ctx_group.chunks[0].blocks for n in G.names]
    check(_unblock(ch.w_stack), *stacked(names))


@pytest.mark.parametrize("pred", [0, 1])
@pytest.mark.parametrize("g", [1.0, 7.5])
def test_sample_step_matches_float64(cuda, pred, g):
    from pcm_b200 import ops, sampling
    B, per = 3, 4 * 16 * 16
    gen = torch.Generator().manual_seed(3)
    cfg = g > 1
    eps = torch.randn(2 * B if cfg else B, per, generator=gen)
    x = torch.randn(B, per, generator=gen)
    coefs = sampling.step_coefficients(sampling.sd15_alphas_cumprod(), 4)
    for _, sa, ss, sap, ssp in (coefs[0], coefs[-1]):     # the last step has prev < 0 (alpha_cumprod[0])
        out = torch.empty(B, per, device=cuda)
        out2 = torch.empty_like(out)
        gb = torch.tensor([g], dtype=torch.float64, device=cuda) if cfg else None
        ops.sample_step(eps.to(cuda), x.to(cuda), out, out2, gb, sa, ss, sap, ssp, pred)
        e = eps.double()
        e = e[:B] + g * (e[B:] - e[:B]) if cfg else e
        xd = x.double()
        x0, pe = ((xd - ss * e) / sa, e) if pred == 0 else (sa * xd - ss * e, sa * e + ss * xd)
        ref = sap * x0 + ssp * pe
        rel = ((out.double().cpu() - ref).norm() / ref.norm()).item()
        assert rel <= 1e-6, rel
        assert torch.equal(out, out2)
    assert coefs[-1][0] - 1000 // 4 < 0


def test_fused_forward_matches_unfused_lora_forward_sd15(cuda):
    """Fused weights (W + s B A rounded once to bf16) against the trained network's unfused LoRA forward
    (bf16 W, bf16 A and s B, bf16 T = x A^T): both are bf16 evaluations of the same function, so their
    distance is the bf16 rounding noise of the network, of the order of DESIGN section 4's distances."""
    from pcm_b200 import config, weights
    from pcm_b200.sampling import PCMSampler
    from pcm_b200.unet import UNetB200
    cfg = config.SD15
    net = UNetB200(cfg, weights.synthetic_state_dict(cfg, 0), cuda, need_backward=False)
    s = PCMSampler(net)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 64, 64, 4, generator=g).to(cuda)
    t = torch.tensor([999, 499], device=cuda)
    ctx = torch.randn(2 * 77, 768, generator=g).to(cuda, BF)
    a = net.forward(x, t, ctx, lora=True)
    b = s.net.forward(x, t, ctx, lora=False)
    base = net.forward(x, t, ctx, lora=False)
    torch.cuda.synchronize()
    rel = ((a - b).double().norm() / a.double().norm()).item()
    lora_part = ((a - base).double().norm() / a.double().norm()).item()
    print(f"fused vs unfused rel-L2 {rel:.3e} (LoRA contribution {lora_part:.3e})")
    assert rel < 2e-2, rel
    assert rel < 0.5 * lora_part            # the fused net carries the adapter, not the base network
    del s, net
    _free()


def _oracle_inputs(ocfg, P, hw):
    g = torch.Generator().manual_seed(11)
    pe = torch.randn(P, 77, ocfg.cross_attention_dim, generator=g)
    ne = torch.randn(P, 77, ocfg.cross_attention_dim, generator=g)
    kw = {}
    if getattr(ocfg, "addition_embed", False):
        kw = dict(text_embeds=torch.randn(P, ocfg.text_embed_dim, generator=g),
                  negative_text_embeds=torch.zeros(P, ocfg.text_embed_dim),
                  time_ids=torch.tensor([hw * 8, hw * 8, 0, 0, hw * 8, hw * 8]))
    return pe, ne, kw


@pytest.mark.parametrize("cfg_name", ["TINY", "TINY_XL"])
def test_sampler_matches_oracle_graph_and_eager(cuda, cfg_name):
    from oracle import unet_ref
    from pcm_b200 import config
    from pcm_b200.sampling import PCMSampler
    from pcm_b200.unet import UNetB200
    ocfg = getattr(unet_ref, cfg_name)
    Pw = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    net = UNetB200(getattr(config, cfg_name), Pw, cuda, need_backward=False)
    s = PCMSampler(net)
    P, nipp, hw = 2, 2, 16
    pe, ne, kw = _oracle_inputs(ocfg, P, hw)
    rep = lambda t: t.repeat_interleave(nipp, 0)  # noqa: E731
    addc = nadd = None
    if kw:
        tid = kw["time_ids"].reshape(1, -1).expand(P * nipp, -1)
        addc = dict(text_embeds=rep(kw["text_embeds"]), time_ids=tid)
        nadd = dict(text_embeds=rep(kw["negative_text_embeds"]), time_ids=tid)
    for n in (1, 2, 4):
        for g in (1.0, 7.5):
            call = dict(num_inference_steps=n, guidance_scale=g, num_images_per_prompt=nipp, height=8 * hw,
                        width=8 * hw, **kw)
            r1 = s(pe, ne, generator=torch.Generator(device=cuda).manual_seed(7), **call)
            r2 = s(pe, ne, generator=torch.Generator(device=cuda).manual_seed(7), **call)   # replay
            assert torch.equal(r1, r2)
            lat = torch.randn(P * nipp, 4, hw, hw, generator=torch.Generator(device=cuda).manual_seed(7), device=cuda)
            s._graphs = False
            e = s(pe, ne, latents=lat, **call)                                                # eager
            s._graphs = True
            assert torch.equal(e, r1), (n, g)
            ref = sample_ref(ocfg, Pw, rep(pe), rep(ne), num_inference_steps=n, latents=lat.cpu(), guidance_scale=g,
                             added_cond=addc, negative_added_cond=nadd, emulate_bf16=True)
            rel = ((r1.cpu().double() - ref.double()).norm() / ref.double().norm()).item()
            assert rel < (2e-2 if g <= 1 else 5e-2), (n, g, rel)
    del s, net
    _free()


def test_sampling_does_not_disturb_training(cuda):
    from pcm_b200 import config, ops, weights
    from pcm_b200.sampling import PCMSampler
    from pcm_b200.step import PCMTrainStep
    cfg = config.TINY
    ops.deterministic(True, cuda)
    try:
        sd = weights.synthetic_state_dict(cfg, 2)
        g = torch.Generator().manual_seed(1)
        B, hw = 2, 16
        inp = (torch.randn(B, hw, hw, 4, generator=g), torch.randn(B, hw, hw, 4, generator=g),
               torch.tensor([3, 30]), torch.tensor([4.5, 4.2]), torch.randn(B, 77, 64, generator=g).to(BF),
               torch.randn(B, 77, 64, generator=g).to(BF))
        res = []
        for sample in (False, True):
            st = PCMTrainStep(cfg, sd, cuda, batch=B, height=hw, width=hw, multiphase=4, lr=1e-3)
            st.load_inputs(*inp)
            st.capture(warmup=1)
            st.step()
            if sample:
                sp = PCMSampler(st.unet)
                opnd = st.unet.lora_opnd.clone()
                for gs in (1.0, 7.5):
                    sp(torch.randn(1, 77, 64), torch.randn(1, 77, 64), num_inference_steps=4, guidance_scale=gs,
                       num_images_per_prompt=4, height=256, width=256)
                torch.cuda.synchronize()
                assert torch.equal(opnd, st.unet.lora_opnd)
            st.step()
            torch.cuda.synchronize()
            res.append([st.loss.clone(), st.unet.lora_master.clone(), st.exp_avg.clone(), st.exp_avg_sq.clone()])
            del st
            _free()
        for a, b in zip(*res):
            assert torch.equal(a, b)
    finally:
        ops.deterministic(False)


def test_cli_validation_end_to_end(cuda, tmp_path):
    from pcm_b200 import config, ops, train_pcm_lora_sd15 as T
    P = 2
    vf = tmp_path / "val.pt"
    torch.save({"prompt_embeds": torch.randn(P, 77, 64, generator=torch.Generator().manual_seed(0))}, vf)
    ops.deterministic(True, cuda)

    def run(out, steps, resume=None, val=True):
        argv = ["--synthetic", "--output_dir", str(out), "--train_batch_size", "2", "--resolution", "128",
                "--multiphase", "4", "--seed", "5", "--learning_rate", "1e-3", "--max_train_steps", str(steps),
                "--checkpointing_steps", "2", "--log_every", "1", "--validation_steps", "2"]
        if val:
            argv += ["--validation_prompt_embeds", str(vf)]
        if resume:
            argv += ["--resume_from_checkpoint", resume]
        a = T.parse_args(argv)
        a._cfg = config.TINY
        st = T.main(a)
        sd = st.state_dict()
        del st
        _free()
        return sd

    try:
        full = run(tmp_path / "a", 4)
        for step in (2, 4):
            for g in (1.0, 7.5):
                d = torch.load(tmp_path / "a" / "validation" / f"step-{step}" / f"cfg-{g}.pt")
                assert d["latents"].shape == (4 * P, 4, 16, 16) and torch.isfinite(d["latents"]).all()
                assert d["seed"] == 5
        run(tmp_path / "b", 2)
        resumed = run(tmp_path / "b", 4, resume="latest")
        plain = run(tmp_path / "c", 4, val=False)
        assert not (tmp_path / "c" / "validation").exists()
        for k in ("lora_master", "exp_avg", "exp_avg_sq"):
            assert torch.equal(full[k], resumed[k]) and torch.equal(full[k], plain[k]), k
        a4 = torch.load(tmp_path / "a" / "validation" / "step-4" / "cfg-7.5.pt")["latents"]
        b4 = torch.load(tmp_path / "b" / "validation" / "step-4" / "cfg-7.5.pt")["latents"]
        assert torch.equal(a4, b4)
    finally:
        ops.deterministic(False)
