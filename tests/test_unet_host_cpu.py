"""HOST logic of pcm_b200/unet.py executed on CPU: every `ops` wrapper is replaced by its torch semantics
(tests/ops_interp.py, tests/gemm_interp.py - descriptors interpreted through their raw pointers), the
sequencing code itself (tape, backward walk, grouped layers, context chunks, merged student + teacher
pass, flat gradient buffer) is the product's.  Compared with the oracle network (oracle/unet_ref.py) on
identical seeded weights - the CPU twin of tests/test_unet_gpu.py (which checks the same with the CUDA
kernels behind the wrappers)."""
import pytest
import torch

import ops_interp
from gemm_interp import BF16, build_net, refresh_operands


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _setup(cfg_name, B, hw, seed=0):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    ocfg = getattr(unet_ref, cfg_name)
    P = unet_ref.init_params(ocfg, seed, lora_b_std=0.02)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=seed)
    net, _ = build_net(getattr(config, cfg_name), sd=P)
    return ocfg, P, batch, net


def _added(ocfg, batch, B):
    if not getattr(ocfg, "addition_embed", False):
        return None, None
    return (batch["text_embeds"], batch["time_ids"]), dict(text_embeds=batch["text_embeds"], time_ids=batch["time_ids"])


@pytest.mark.parametrize("cfg_name", ["TINY", "TINY_XL"])
def test_forward_and_backward_match_the_oracle(monkeypatch, cfg_name):
    from oracle import unet_ref
    B, hw = 2, 8
    ocfg, P, batch, net = _setup(cfg_name, B, hw)
    ops_interp.install(monkeypatch)
    x, ctx = batch["latents"], batch["prompt_embeds"]
    ts = torch.tensor([999, 19])
    added, okw = _added(ocfg, batch, B)
    kw = {} if okw is None else dict(added_cond_kwargs=okw)
    ctx2 = ctx.to(BF16).reshape(B * ctx.shape[1], -1)
    for lora in (True, False):
        ref = unet_ref.UNetRef(ocfg, P, use_lora=lora, emulate_bf16=True)(x, ts, ctx, **kw)
        out = _nchw(net.forward(_nhwc(x), ts, ctx2, lora=lora, added_cond=added))
        err = (out - ref).abs()
        assert err.max().item() <= 3e-2 * ref.abs().max().item(), (lora, err.max().item())
        assert err.mean().item() <= 1e-2 * ref.pow(2).mean().sqrt().item(), (lora, err.mean().item())
    # backward: LoRA gradients of sum(eps * G)
    G = torch.randn(B, 4, hw, hw, generator=torch.Generator().manual_seed(7)) / (B * 4 * hw * hw)
    Pg = {k: (v.clone().requires_grad_(True) if ".lora_" in k else v) for k, v in P.items()}
    eps = unet_ref.UNetRef(ocfg, Pg, use_lora=True, emulate_bf16=True)(x, ts, ctx, **kw)
    (eps * G).sum().backward()
    net.forward(_nhwc(x), ts, ctx2, lora=True, save=True, added_cond=added)
    net.lora_grad.zero_()
    net.backward(_nhwc(G))
    g = net.lora_grad_dict()
    num = den = 0.0
    for k, v in Pg.items():
        if ".lora_" in k:
            num += (g[k].float() - v.grad.reshape(g[k].shape)).pow(2).sum().item()
            den += v.grad.pow(2).sum().item()
    assert (num / den) ** 0.5 <= 5e-2, (num / den) ** 0.5


def test_merged_pass_equals_student_plus_frozen_teacher(monkeypatch):
    """lora_batch = b < B: the leading b samples see the adapter, the others the frozen network, in ONE
    pass; the tape then belongs to the student samples and backward() gives the student's gradients."""
    B, hw = 3, 8
    ocfg, P, batch, net = _setup("TINY", B, hw)
    ops_interp.install(monkeypatch)
    x, ctx = _nhwc(batch["latents"]), batch["prompt_embeds"].to(BF16)
    S = ctx.shape[1]
    ctx2 = ctx.reshape(B * S, -1)
    ts = torch.tensor([999, 19, 499])
    merged = net.forward(x, ts, ctx2, lora=True, save=True, lora_batch=1)
    kv = net.saved_ctx_kv()
    G = torch.randn(1, hw, hw, 4, generator=torch.Generator().manual_seed(8)) / (4 * hw * hw)
    net.lora_grad.zero_()
    net.backward(G)
    g_merged = net.lora_grad.clone()
    stu = net.forward(x[:1], ts[:1], ctx2[:S], lora=True, save=True)
    net.lora_grad.zero_()
    net.backward(G)
    tea = net.forward(x[1:], ts[1:], ctx2[S:], lora=False)
    assert torch.equal(merged[:1], stu) and torch.equal(merged[1:], tea)
    # (same launches on the same student rows; torch's CPU matmul blocking may differ in the last bit)
    assert ((g_merged - net.lora_grad).norm() / net.lora_grad.norm()).item() < 1e-5 and g_merged.abs().max() > 0
    # the target pass of the step takes the student rows of the merged pass's context projections
    sub = net.ctx_kv_rows(kv, S)
    again = net.forward(x[:1], ts[:1], ctx2[:S], lora=True, ctx_kv=sub)
    assert torch.equal(again, stu)


VARIANTS = {
    "reference": dict(),
    "v_prediction_l2": dict(prediction_type="v_prediction", loss_type="l2"),
    "no_cfg_solver": dict(apply_cfg_solver=False),
    "two_substeps": dict(teacher_substeps=2),
    "two_phases": dict(multiphase=2),
    "ema_target": dict(ema_decay=0.95),      # EMA copy == student at step 0: same numbers, other code path
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_step_host_sequence_matches_the_oracle_iteration(monkeypatch, variant):
    """PCMTrainStep.forward_backward on CPU (every kernel replaced by its torch semantics): merged student +
    teacher pass, teacher DDIM step, target pass on the student's context projections, loss, backward -
    vs oracle/pcm_ref.pcm_step_ref (T15:1139-1296).  CPU twin of
    tests/test_unet_gpu.py::test_step_loss_and_grads_match_oracle."""
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, ops
    from pcm_b200.step import PCMTrainStep
    kw =dict(VARIANTS[variant])
    B, hw, multiphase = 2, 8, kw.pop("multiphase", 4)
    ocfg = unet_ref.TINY
    P = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=0)
    okw = {k: v for k, v in kw.items() if k != "ema_decay"}
    ref = pcm_ref.pcm_step_ref(ocfg, P, batch, multiphase=multiphase, emulate_bf16=True, need_grad=True, **okw)
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        st = PCMTrainStep(config.TINY, P, "cpu", batch=B, height=hw, width=hw, multiphase=multiphase,
                          keep_debug=True, **kw)
    finally:
        ops.DRY_RUN = old
    net = st.unet
    refresh_operands(net)
    ops_interp.install_step(monkeypatch)
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF16), batch["uncond_prompt_embeds"].to(BF16))
    net.lora_grad.zero_()
    st.forward_backward()
    assert torch.equal(st.start_t, ref["start_timesteps"]) and torch.equal(st.t, ref["timesteps"])
    assert torch.equal(st.end_t, ref["end_timesteps"])
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()  # noqa: E731
    assert rel(_nchw(st.debug["eps_student"]), ref["eps_student"]) < 2e-2
    # v_prediction: x_prev = sqrt(a')(a x - s v) + sqrt(1-a') v does not cancel the bf16 noise of the
    # CFG-amplified teacher output the way the epsilon form does (the kernels themselves: 1e-6,
    # tests/test_pcm_kernels_gpu.py)
    tol = 1.5e-1 if kw.get("prediction_type") == "v_prediction" else 2e-2
    assert rel(_nchw(st.x_prev), ref["x_prev"]) < tol
    assert rel(_nchw(st.model_pred), ref["model_pred"]) < tol and rel(_nchw(st.target), ref["target"]) < tol
    assert abs(st.loss.item() - ref["loss"].item()) <= 4e-2 * ref["loss"].item()
    g = net.lora_grad_dict()
    dot = n1 = n2 = 0.0
    for k, rg in ref["grads"].items():
        gg = g[k].float().reshape(rg.shape)
        dot += (gg * rg).sum().item()
        n1 += gg.pow(2).sum().item()
        n2 += rg.pow(2).sum().item()
    cos = dot / (n1 ** 0.5 * n2 ** 0.5)
    print(f"[host step, {variant}] loss {st.loss.item():.6f} (oracle {ref['loss'].item():.6f}) | rel-L2 eps "
          f"{rel(_nchw(st.debug['eps_student']), ref['eps_student']):.2e} x_prev {rel(_nchw(st.x_prev), ref['x_prev']):.2e} "
          f"| LoRA-gradient cosine {cos:.4f}")
    assert cos >= 0.85          # same bound as the GPU twin (Huber sign noise)


def test_sdxl_shaped_step_host_sequence(monkeypatch):
    """SDXL-shaped network through the whole step on CPU: 40 DDIM steps, added conditions (pooled text
    embedding + time ids) on every pass, ZERO unconditional embeddings, transformer depth (1, 2, 3) -
    train_pcm_lora_sdxl_adv.py:1094-1133, 1215-1221.  CPU twin of tests/test_sdxl_gpu.py::test_sdxl_step_loss."""
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, ops
    from pcm_b200.step import PCMTrainStep
    B, hw, mp = 2, 8, 4
    ocfg = unet_ref.TINY_XL
    P = unet_ref.init_params(ocfg, 1)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=1, num_ddim=40, zero_uncond=True)
    ref = pcm_ref.pcm_step_ref(ocfg, P, batch, multiphase=mp, num_ddim=40, emulate_bf16=True, need_grad=False)
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        st = PCMTrainStep(config.TINY_XL, P, "cpu", batch=B, height=hw, width=hw, multiphase=mp,
                          num_ddim_timesteps=40, keep_debug=True)
    finally:
        ops.DRY_RUN = old
    refresh_operands(st.unet)
    ops_interp.install_step(monkeypatch)
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF16), batch["uncond_prompt_embeds"].to(BF16),
                   text_embeds=batch["text_embeds"].to(BF16), time_ids=batch["time_ids"])
    st.forward_backward()
    assert torch.equal(st.start_t, ref["start_timesteps"]) and torch.equal(st.end_t, ref["end_timesteps"])
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()  # noqa: E731
    assert rel(_nchw(st.x_prev), ref["x_prev"]) < 2e-2 and rel(_nchw(st.model_pred), ref["model_pred"]) < 2e-2
    assert abs(st.loss.item() - ref["loss"].item()) <= 4e-2 * ref["loss"].item()
    assert st.unet.lora_grad.abs().max() > 0
