"""LoRA ranks other than 64 on the H100 kernels: narrow K chunks of pcm_gemm, narrow and multiple rank
slices of pcm_wgrad, pcm_lora_refresh at any rank, and the UNet / step against the CPU oracle."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rand(shape, dev, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(torch.bfloat16)


def _pad64(t):
    return F.pad(t, (0, 64 * ((t.shape[-1] + 63) // 64) - t.shape[-1]))


@pytest.mark.parametrize("r", [8, 16, 32, 48, 96])
def test_gemm_narrow_lora_chunk_equals_zero_padded(cuda, r):
    """Base K blocks + a LoRA up-projection chunk of width r: bitwise the same GEMM with T and s*B
    zero-padded to whole 64-column chunks in memory, and close to fp32 torch."""
    from pcm_b200 import ops
    M, K, N = 1000, 320, 192
    x, w = _rand((M, K), cuda, 1), _rand((N, K), cuda, 2, K ** -0.5)
    T, sb = _rand((M, r), cuda, 3), _rand((N, r), cuda, 4, 0.05)
    nc = (r + 63) // 64
    outs = []
    for TT, SB in ((T, sb), (_pad64(T), _pad64(sb))):
        out = torch.empty(M, N, device=cuda, dtype=torch.bfloat16)
        ops.gemm([ops.asrc_mat(x), ops.asrc_mat(TT)], [ops.bsrc(w), ops.bsrc(SB)],
                 [(0, 0, 0, 0, K // 64, 0, 0), (1, 1, 0, 0, nc, 0, 0)], lin=True, M=M, N=N, out=out)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    ref = x.float() @ w.float().t() + T.float() @ sb.float().t()
    err = (outs[0].float() - ref).abs()
    assert err.max().item() <= 1e-2 * ref.abs().max().item()


@pytest.mark.parametrize("r", [8, 32, 48])
def test_gemm_stacked_T_and_conv_dgrad_taps(cuda, r):
    """Grouped layers: N-ranged LoRA entries reading column blocks i*r of a stacked T against s*B (K = r),
    and a conv dgrad's LoRA entries (dt, C = r) against A^T at b_k0 = t*r."""
    from pcm_b200 import ops
    M, K, C, g = 512, 128, 96, 3
    x, w = _rand((M, K), cuda, 1), _rand((g * C, K), cuda, 2, K ** -0.5)
    T, sb = _rand((M, g * r), cuda, 3), _rand((g * C, r), cuda, 4, 0.05)
    out = torch.empty(M, g * C, device=cuda, dtype=torch.bfloat16)
    prog = [(0, 0, 0, 0, K // 64, 0, 0)] + [(1, 1, 0, 0, 1, i * r, 0, i * C, (i + 1) * C) for i in range(g)]
    ops.gemm([ops.asrc_mat(x), ops.asrc_mat(T)], [ops.bsrc(w), ops.bsrc(sb)], prog, lin=True, M=M, N=g * C,
             out=out, block_n=32)
    ref = x.float() @ w.float().t()
    for i in range(g):
        ref[:, i * C:(i + 1) * C] += T[:, i * r:(i + 1) * r].float() @ sb[i * C:(i + 1) * C].float().t()
    err = (out.float() - ref).abs()
    assert err.max().item() <= 1e-2 * ref.abs().max().item()
    # conv dgrad LoRA taps: dx[m, c] = sum_t dt[m - tap t, :] . a_t[c, t*r:(t+1)*r]
    B, H, W, cin = 2, 16, 16, 64
    dt = _rand((B, H, W, r), cuda, 5)
    a_t = _rand((cin, 9 * r), cuda, 6, 0.1)
    dx = torch.empty(B * H * W, cin, device=cuda, dtype=torch.float32)
    prog = [(0, 0, -dw, -dh, 1, 0, t * r) for t, (dw, dh) in enumerate(ops.TAPS3)]
    ops.gemm([ops.asrc_nhwc(dt)], [ops.bsrc(a_t)], prog, lin=False, M=B * H * W, N=cin, geo=(W, H), out=dx)
    wconv = a_t.float().view(cin, 3, 3, r).permute(0, 3, 1, 2)      # [cin, r, kh, kw] of the forward A
    ref = F.conv_transpose2d(dt.float().permute(0, 3, 1, 2), wconv.permute(1, 0, 2, 3), padding=1)
    got = dx.view(B, H, W, cin).permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


@pytest.mark.parametrize("width,slices", [(8, 1), (32, 1), (48, 1), (128, 2)])
def test_wgrad_narrow_and_multiple_slices(cuda, width, slices):
    """dB[ch, r] += s * P^T Q for a rank slice narrower than 64 (and two slices at r = 128): fp32 torch
    parity, NaN sentinels around the gradient and in the neighbouring layer's rows stay untouched, and the
    deterministic mode is bit-identical over repeated launches."""
    from pcm_b200 import ops
    M, Cp, r = 1000, 192, width
    p = _rand((M, Cp), cuda, 1)
    qs = _rand((M, 3 * r), cuda, 2)      # stacked: this layer's ranks are columns [r, 2r)
    ref = 0.25 * p.float().t() @ qs[:, r:2 * r].float()
    results = []
    for det in (False, True, True):
        ops.deterministic(det, cuda)
        buf = torch.full((Cp * r + 2 * 64,), float("nan"), device=cuda)
        gB = buf[64:64 + Cp * r].view(Cp, r)
        gB.zero_()
        q = ops.asrc_cols(ops.asrc_mat(qs), 2 * r) if r % 64 else ops.asrc_mat(qs)
        for j in range(slices):
            ops.wgrad(ops.asrc_mat(p), q, gB[:, 64 * j:], lin=True, M=M, os_row=r, os_col=1, alpha=0.25,
                      q_c0=r + 64 * j)
        torch.cuda.synchronize()
        assert torch.isnan(buf[:64]).all() and torch.isnan(buf[64 + Cp * r:]).all()
        assert (gB - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()
        results.append(gB.clone())
    ops.deterministic(False)
    assert torch.equal(results[1], results[2])
    # transposed destination (dA layout [r, cin]): rows past the slice belong to the next layer
    gA_buf = torch.full((r + 8, Cp), float("nan"), device=cuda)
    gA = gA_buf[:r]
    gA.zero_()
    q = ops.asrc_mat(qs[:, :r].contiguous())
    for j in range(slices):
        ops.wgrad(ops.asrc_mat(p), q, gA[64 * j:], lin=True, M=M, os_row=1, os_col=Cp, q_c0=64 * j)
    torch.cuda.synchronize()
    assert torch.isnan(gA_buf[r:]).all()
    refA = (p.float().t() @ qs[:, :r].float()).t()
    assert (gA - refA).abs().max().item() <= 2e-3 * refA.abs().max().item()


@pytest.mark.parametrize("r", [8, 32, 48, 128])
def test_lora_refresh_any_rank(cuda, r):
    from pcm_b200 import config, weights
    from pcm_b200.unet import UNetB200
    cfg = dataclasses.replace(config.TINY, lora_rank=r)
    sd = weights.synthetic_state_dict(cfg, 0, lora_b_std=0.2)
    net = UNetB200(cfg, sd, cuda, lora=True, need_backward=True)
    net.lora_opnd.fill_(float("nan"))
    net.refresh_lora()
    torch.cuda.synchronize()
    assert not torch.isnan(net.lora_opnd.float()).any()
    for L in net.lora_layers:
        lo = L.lora
        taps = L.k * L.k if L.kind == "conv" else 1
        A = net.lora_master[lo.a_off:lo.a_off + r * taps * L.cin].view(r, taps * L.cin).to(torch.bfloat16)
        sB = (net.scale * net.lora_master[lo.b_off:lo.b_off + L.cout * r].view(L.cout, r)).to(torch.bfloat16)
        assert torch.equal(lo.a_fwd, A) and torch.equal(lo.sb_fwd, sB) and torch.equal(lo.sb_t, sB.t())
        assert torch.equal(lo.a_t, A.view(r, taps, L.cin).permute(2, 1, 0).reshape(L.cin, taps * r))


@pytest.mark.parametrize("r", [8, 32, 128])
def test_step_matches_the_oracle_at_rank(cuda, r):
    """The whole step (loss, LoRA gradients, clip + AdamW) at rank r vs the CPU oracle, with the
    tolerances of tests/test_unet_gpu.py."""
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    from pcm_b200.step import PCMTrainStep
    B, hw, mp = 2, 16, 4
    ocfg = dataclasses.replace(unet_ref.TINY, lora_rank=r)
    P = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=0)
    ref = pcm_ref.pcm_step_ref(ocfg, P, batch, multiphase=mp, emulate_bf16=True, need_grad=True)
    st = PCMTrainStep(dataclasses.replace(config.TINY, lora_rank=r), P, cuda, batch=B, height=hw, width=hw,
                      multiphase=mp)
    nhwc = lambda x: x.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    st.load_inputs(nhwc(batch["latents"]), nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].bfloat16(), batch["uncond_prompt_embeds"].bfloat16())
    st.unet.lora_grad.zero_()
    st.forward_backward()
    torch.cuda.synchronize()
    assert abs(st.loss.item() - ref["loss"].item()) <= 4e-2 * ref["loss"].item()
    g = st.unet.lora_grad_dict()
    dot = n1 = n2 = 0.0
    for k, rg in ref["grads"].items():
        gg = g[k].float().cpu().reshape(rg.shape)
        dot += (gg * rg).sum().item()
        n1 += gg.pow(2).sum().item()
        n2 += rg.pow(2).sum().item()
    assert dot / (n1 ** 0.5 * n2 ** 0.5) >= 0.85
    before = st.unet.lora_master.clone()
    st.optimizer_step()
    torch.cuda.synchronize()
    assert torch.isfinite(st.unet.lora_master).all() and not torch.equal(before, st.unet.lora_master)


def test_checkpointed_step_is_the_stored_tape_at_rank_32(cuda):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, ops
    from pcm_b200.step import PCMTrainStep
    B, hw, mp, r = 2, 16, 4, 32
    ocfg = dataclasses.replace(unet_ref.TINY, lora_rank=r)
    P = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=0)
    nhwc = lambda x: x.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    ops.deterministic(True, cuda)
    try:
        grads = []
        for ck in (False, True):
            st = PCMTrainStep(dataclasses.replace(config.TINY, lora_rank=r), P, cuda, batch=B, height=hw,
                              width=hw, multiphase=mp, gradient_checkpointing=ck)
            st.load_inputs(nhwc(batch["latents"]), nhwc(batch["noise"]), batch["index"], batch["w"],
                           batch["prompt_embeds"].bfloat16(), batch["uncond_prompt_embeds"].bfloat16())
            st.unet.lora_grad.zero_()
            st.forward_backward()
            torch.cuda.synchronize()
            grads.append((st.loss.clone(), st.unet.lora_grad.clone()))
        assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    finally:
        ops.deterministic(False)


def _cli(tmp, extra):
    from pcm_b200 import config, train_pcm_lora_sd15 as T
    argv = ["--synthetic", "--output_dir", str(tmp), "--train_batch_size", "2", "--resolution", "128",
            "--multiphase", "4", "--seed", "5", "--checkpointing_steps", "2", "--log_every", "1"] + list(extra)
    a = T.parse_args(argv)
    a._cfg = dataclasses.replace(config.TINY, lora_rank=a.lora_rank)
    return T, a


def test_cli_trains_and_resumes_at_rank_32(cuda, tmp_path):
    """--lora_rank 32 trains, writes rank-32 artefacts, resumes to the parameters of an uninterrupted run;
    resuming that checkpoint with --lora_rank 64 raises."""
    import json
    from safetensors.torch import load_file
    from pcm_b200 import ops
    ops.deterministic(True, cuda)
    try:
        T, a = _cli(tmp_path / "straight", ["--lora_rank", "32", "--max_train_steps", "4"])
        full = T.main(a).unet.lora_master.clone()
        T, a = _cli(tmp_path / "resumed", ["--lora_rank", "32", "--max_train_steps", "2"])
        T.main(a)
        out = tmp_path / "resumed"
        cfgj = json.load(open(out / "adapter_config.json"))
        assert cfgj["r"] == 32 and cfgj["lora_alpha"] == 8
        sd = load_file(str(out / "adapter_model.safetensors"))
        assert sd and all(v.shape[0] == 32 for k, v in sd.items() if "lora_A" in k)
        assert all(v.shape[1] == 32 for k, v in sd.items() if "lora_B" in k)
        T, a = _cli(out, ["--lora_rank", "64", "--max_train_steps", "4", "--resume_from_checkpoint", "latest"])
        with pytest.raises(ValueError, match="rank-32"):
            T.main(a)
        T, a = _cli(out, ["--lora_rank", "32", "--max_train_steps", "4", "--resume_from_checkpoint", "latest"])
        st = T.main(a)
        assert torch.equal(st.unet.lora_master, full)
    finally:
        ops.deterministic(False)
