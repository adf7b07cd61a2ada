"""The BASELINE configurations through the product's HOST code on CPU (SD1.5-width UNet, 278 LoRA layers,
merged batch-3B pass, context chunks, explicit backward), every kernel replaced by its torch semantics
(tests/ops_interp.py), against the golden vectors of the oracle step (tests/golden/step_config{1,2}.pt) -
the CPU twin of tests/test_parity_gpu.py.  What it shows: the launch PLAN of the benchmark network is the
reference iteration; what it cannot show: the CUDA kernels (that is the GPU twin's job).

config 1 (bs 1, 32x32, 2-phase) runs in ~20 s; config 2 (bs 8, 64x64, 4-phase, the benchmark workload)
needs several minutes of CPU and runs only with PCM_SLOW_TESTS=1 (measured numbers: DESIGN.md section 4)."""
import os

import pytest
import torch

import ops_interp
from gemm_interp import refresh_operands

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BF16 = torch.bfloat16


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _at(g, x):
    """x (NCHW) at the positions the golden file stores: all, or the fixed sample `sample_idx` (config 2)."""
    idx = g.get("sample_idx")
    return x if idx is None else x.reshape(-1)[idx.long()]


def _run(monkeypatch, c):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, ops
    from pcm_b200.step import PCMTrainStep
    g = torch.load(os.path.join(GOLD, f"step_config{c}.pt"))
    B, hw, mp = g["config"]["B"], g["config"]["hw"], g["config"]["multiphase"]
    P = unet_ref.init_params(unet_ref.SD15, 0)
    batch = pcm_ref.make_batch(unet_ref.SD15, B, hw, seed=0)
    assert torch.equal(batch["index"], g["index"]) and torch.equal(batch["w"], g["w"])
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        st = PCMTrainStep(config.SD15, P, "cpu", batch=B, height=hw, width=hw, multiphase=mp, lr=5e-6,
                          weight_decay=1e-3, keep_debug=True)
    finally:
        ops.DRY_RUN = old
    refresh_operands(st.unet)
    ops_interp.install_step(monkeypatch)
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF16), batch["uncond_prompt_embeds"].to(BF16))
    st.forward_backward()
    r = g["bf16"]
    assert torch.equal(st.start_t, r["start_timesteps"]) and torch.equal(st.t, r["timesteps"])
    assert torch.equal(st.end_t, r["end_timesteps"])
    assert torch.equal(_at(g, _nchw(st.noisy)), r["noisy"])                     # add_noise: bit-exact op sequence
    rows = {}
    for mode in ("bf16", "fp32"):
        r = g[mode]
        rows[mode] = dict(loss=abs(st.loss.item() - r["loss"].item()) / r["loss"].item(),
                          eps=_rel(_at(g, _nchw(st.debug["eps_student"])), r["eps_student"]),
                          x_prev=_rel(_at(g, _nchw(st.x_prev)), r["x_prev"]),
                          model_pred=_rel(_at(g, _nchw(st.model_pred)), r["model_pred"]),
                          target=_rel(_at(g, _nchw(st.target)), r["target"]))
        print(f"[host parity config {c}] vs {mode} oracle: loss {st.loss.item():.8f} (oracle {r['loss'].item():.8f}) "
              f"rel {rows[mode]['loss']:.3e} | rel-L2 eps {rows[mode]['eps']:.3e} x_prev {rows[mode]['x_prev']:.3e} "
              f"model_pred {rows[mode]['model_pred']:.3e} target {rows[mode]['target']:.3e}", flush=True)
    g_norm = st.unet.lora_grad.norm().item()
    assert g_norm > 0 and torch.isfinite(st.unet.lora_grad).all()
    return rows


def test_config1_host_plan_matches_golden(monkeypatch):
    rows = _run(monkeypatch, 1)
    # same bounds as the GPU twin (tests/test_parity_gpu.py)
    assert rows["bf16"]["loss"] <= 1.5e-2 and rows["fp32"]["loss"] <= 2e-2
    for k in ("eps", "x_prev", "model_pred", "target"):
        assert rows["bf16"][k] <= 3e-2 and rows["fp32"][k] <= 6e-2, (k, rows)


@pytest.mark.skipif(os.environ.get("PCM_SLOW_TESTS", "0") != "1", reason="several CPU minutes: PCM_SLOW_TESTS=1")
def test_config2_host_plan_matches_golden(monkeypatch):
    rows = _run(monkeypatch, 2)
    assert rows["bf16"]["loss"] <= 2e-3 and rows["fp32"]["loss"] <= 1.2e-2
    for k in ("eps", "x_prev", "model_pred", "target"):
        assert rows["bf16"][k] <= 3e-2 and rows["fp32"][k] <= 6e-2, (k, rows)


def test_sd15_width_backward_plan_vs_oracle_autograd(monkeypatch):
    """LoRA gradients of sum(eps * G) for a fixed cotangent G at SD1.5 width (all 278 adapters, bs 1, 32x32):
    the product's explicit backward walk (dgrad K programs, 1112 weight-gradient launches into the flat
    buffer) vs torch autograd through the oracle network."""
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    from gemm_interp import build_net
    B, hw = 1, 32
    P = unet_ref.init_params(unet_ref.SD15, 0)
    batch = pcm_ref.make_batch(unet_ref.SD15, B, hw, seed=0)
    x, ctx = batch["latents"], batch["prompt_embeds"]
    ts = torch.tensor([499])
    G = torch.randn(B, 4, hw, hw, generator=torch.Generator().manual_seed(7)) / (B * 4 * hw * hw)
    Pg = {k: (v.clone().requires_grad_(True) if ".lora_" in k else v) for k, v in P.items()}
    eps = unet_ref.UNetRef(unet_ref.SD15, Pg, use_lora=True, emulate_bf16=True)(x, ts, ctx)
    (eps * G).sum().backward()
    net, _ = build_net(config.SD15, sd=P)
    ops_interp.install(monkeypatch)
    out = net.forward(_nhwc(x), ts, ctx.to(BF16).reshape(B * 77, -1), lora=True, save=True)
    assert _rel(_nchw(out), eps.detach()) <= 3e-2
    net.lora_grad.zero_()
    net.backward(_nhwc(G))
    g = net.lora_grad_dict()
    num = den = 0.0
    worst = 0.0
    n = 0
    for k, v in Pg.items():
        if ".lora_" in k:
            d = (g[k].float() - v.grad.reshape(g[k].shape))
            num += d.pow(2).sum().item()
            den += v.grad.pow(2).sum().item()
            worst = max(worst, (d.norm() / (v.grad.norm() + 1e-20)).item())
            n += 1
    print(f"[host backward SD1.5] {n} LoRA tensors: global rel-L2 {(num / den) ** 0.5:.3e}, worst tensor {worst:.3e}")
    assert n == 2 * 278 and (num / den) ** 0.5 <= 5e-2 and worst <= 0.15
