"""Parity of the WHOLE step at the BASELINE configurations, exactly as bench.py runs it (SD1.5 UNet,
merged batch-3B student + teacher pass, eager AND CUDA-graph replay), against the golden vectors of
the oracle step (tests/golden/step_config{1,2}.pt, written on the CPU by
tests/golden/make_step_golden.py from oracle/pcm_ref.py::pcm_step_ref):

    config 1   bs 1, 32x32 latents, 2-phase   (the reference's CPU smoke configuration)
    config 2   bs 8, 64x64 latents, 4-phase   (the benchmark workload)

Two oracle modes are compared and REPORTED (printed, see DESIGN.md section 4 for the table):
  * `bf16`  - the oracle rounding where bf16 autocast materialises tensors: implementation parity.
              Asserted: loss within LOSS_TOL_BF16, tensors within bf16 accumulation-order noise.
  * `fp32`  - the reference's CPU semantics (fp32 end to end).  The bf16 networks add independent
              rounding noise e to model_pred - target = d, and E|d + e| > E|d| for the Huber loss, so
              a bf16 run (this one, or the reference's own under --mixed_precision=bf16) sits a few
              percent ABOVE the fp32 loss on random-init weights; asserted at LOSS_TOL_FP32 (2x the
              measured value), not at the north-star's 1e-3, which bf16 arithmetic cannot meet here.
Also: bit-reproducibility of repeated steps (deterministic mode) and the run-to-run loss spread
without it.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# see DESIGN.md section 4 for why the fp32-oracle bounds sit above the bf16 ones.
# Config 2 (N = 131072 loss terms): 2.7e-4 and 7.8e-5 on two builds -> 2e-3 (north-star 1e-3 met).
# Config 1 (N = 4096 loss terms only): the loss is a mean of |model_pred - target| over few, noisy terms;
# two builds with IDENTICAL tensor accuracy (rel-L2 eps 8.29e-3 both) measured 3.0e-3 and 6.8e-3 -> 1.5e-2.
LOSS_TOL_BF16 = {1: 1.5e-2, 2: 2e-3}
LOSS_TOL_FP32 = {1: 2e-2, 2: 1.2e-2}
TENSOR_TOL_BF16 = 3e-2       # rel. L2 of eps / x_prev / model_pred / target vs the bf16 oracle
TENSOR_TOL_FP32 = 6e-2


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _at(g, x):
    """x (NCHW, on the CPU) at the positions the golden file stores: all of them, or the fixed sample
    `sample_idx` of flat positions (config 2)."""
    idx = g.get("sample_idx")
    return x if idx is None else x.reshape(-1)[idx.long()]


_CACHE = {}


def _sd15_params():
    """Seeded SD1.5-shaped weights, identical to the ones the golden vectors were made with."""
    if "P" not in _CACHE:
        from oracle import unet_ref
        _CACHE["P"] = unet_ref.init_params(unet_ref.SD15, 0)
    return _CACHE["P"]


def _golden(c):
    path = os.path.join(GOLD, f"step_config{c}.pt")
    if not os.path.exists(path):
        pytest.skip(f"{path} missing: run tests/golden/make_step_golden.py {c}")
    g = torch.load(path)
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_step_golden", os.path.join(GOLD, "make_step_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    chk = m.param_checksum(_sd15_params())
    assert torch.allclose(chk, g["param_checksum"], rtol=1e-12, atol=0), \
        "seeded weights differ from the ones the golden vectors were generated with"
    return g


def _make_step(cuda, c, **kw):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    from pcm_b200.step import PCMTrainStep
    g = _golden(c)
    B, hw, mp = g["config"]["B"], g["config"]["hw"], g["config"]["multiphase"]
    batch = pcm_ref.make_batch(unet_ref.SD15, B, hw, seed=0)
    assert torch.equal(batch["index"], g["index"]) and torch.equal(batch["w"], g["w"])
    st = PCMTrainStep(config.SD15, _sd15_params(), cuda, batch=B, height=hw, width=hw, multiphase=mp,
                      lr=5e-6, weight_decay=1e-3, keep_debug=True, **kw)
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF), batch["uncond_prompt_embeds"].to(BF))
    return g, st


def _report(tag, c, st, g):
    rows = {}
    for mode in ("bf16", "fp32"):
        r = g[mode]
        rows[mode] = dict(
            loss=abs(st.loss.item() - r["loss"].item()) / abs(r["loss"].item()),
            eps_student=_rel(_at(g, _nchw(st.debug["eps_student"]).cpu()), r["eps_student"]),
            x_prev=_rel(_at(g, _nchw(st.x_prev).cpu()), r["x_prev"]),
            model_pred=_rel(_at(g, _nchw(st.model_pred).cpu()), r["model_pred"]),
            target=_rel(_at(g, _nchw(st.target).cpu()), r["target"]))
        print(f"[parity config {c} {tag}] vs {mode} oracle: loss {st.loss.item():.8f} (oracle "
              f"{r['loss'].item():.8f}) rel {rows[mode]['loss']:.3e} | rel-L2 eps {rows[mode]['eps_student']:.3e} "
              f"x_prev {rows[mode]['x_prev']:.3e} model_pred {rows[mode]['model_pred']:.3e} "
              f"target {rows[mode]['target']:.3e}", flush=True)
    return rows


def _check(c, st, g, rows):
    r = g["bf16"]
    assert torch.equal(st.start_t.cpu(), r["start_timesteps"])
    assert torch.equal(st.t.cpu(), r["timesteps"])
    assert torch.equal(st.end_t.cpu(), r["end_timesteps"])
    assert torch.equal(_at(g, _nchw(st.noisy).cpu()), r["noisy"])   # add_noise is bit-exact
    assert rows["bf16"]["loss"] <= LOSS_TOL_BF16[c], rows
    assert rows["fp32"]["loss"] <= LOSS_TOL_FP32[c], rows
    for k in ("eps_student", "x_prev", "model_pred", "target"):
        assert rows["bf16"][k] <= TENSOR_TOL_BF16, (k, rows)
        assert rows["fp32"][k] <= TENSOR_TOL_FP32, (k, rows)


@pytest.mark.parametrize("c", [1, 2])
def test_step_parity_eager_and_graph(cuda, c):
    """Eager step, then the SAME step captured into one CUDA graph and replayed (what bench.py times):
    both against the golden oracle vectors; graph replay must reproduce the eager loss bit for bit."""
    g, st = _make_step(cuda, c)
    st.forward_backward()
    torch.cuda.synchronize()
    rows = _report("eager", c, st, g)
    _check(c, st, g, rows)
    loss_eager = st.loss.item()
    mp_eager = st.model_pred.clone()
    st.unet.lora_grad.zero_()
    st.capture(warmup=1)
    st.step()
    torch.cuda.synchronize()
    rows = _report("graph", c, st, g)
    _check(c, st, g, rows)
    assert st.loss.item() == loss_eager, (st.loss.item(), loss_eager)
    assert torch.equal(st.model_pred, mp_eager)


def test_merged_pass_matches_separate_passes(cuda):
    """The merged batch-3B pass (student + both teacher passes in one forward, LoRA rows TMA-zero
    filled for the teacher samples) against separate forwards of the student (LoRA) and of both
    teacher halves (frozen network): same predictions, x_prev and loss within bf16 noise."""
    g, st = _make_step(cuda, 1)
    st.forward_backward()
    torch.cuda.synchronize()
    merged = [st.debug[k].clone() for k in ("eps_student", "eps_cond", "eps_uncond")]
    l_merged, xp_merged = st.loss.item(), st.x_prev.clone()
    u, B = st.unet, st.B
    eps_s = u.forward(st.noisy, st.start_t, st.in_prompt, lora=True)
    eps_cu = u.forward(st.noisy3[B:], st.start_t3[B:], st.in_ctx3[B * 77:], lora=False)
    st.teacher_step_kernel(eps_cu[:B], eps_cu[B:])
    st.loss_kernel(eps_s, u.forward(st.x_prev, st.t, st.in_prompt, lora=True))
    torch.cuda.synchronize()
    for name, sep, mrg in zip(("student", "cond", "uncond"), (eps_s, eps_cu[:B], eps_cu[B:]), merged):
        assert _rel(sep, mrg) <= 2e-2, (name, _rel(sep, mrg))
    assert _rel(st.x_prev, xp_merged) <= 2e-2
    assert abs(st.loss.item() - l_merged) <= 2e-2 * abs(l_merged)


def test_repeated_steps_bit_identical(cuda):
    """Deterministic mode: 10 repetitions of the same step from the same state give bit-identical
    loss, predictions, LoRA gradients and updated parameters (config 1 exercises split-K, the
    GroupNorm partial merges, the ordered weight-gradient splits and the fixed-order norm)."""
    from pcm_b200 import ops
    ops.deterministic(True, cuda)
    try:
        g, st = _make_step(cuda, 1)
        snap = st.state_dict()
        ref = None
        for i in range(10):
            st.load_state_dict(snap)
            st.run_eager()
            torch.cuda.synchronize()
            cur = (st.loss.clone(), st.model_pred.clone(), st.target.clone(), st.unet.lora_master.clone(),
                   st.exp_avg_sq.clone())
            if ref is None:
                ref = cur
            else:
                for a, b in zip(ref, cur):
                    assert torch.equal(a, b), f"repetition {i} differs"
    finally:
        ops.deterministic(False)


def test_loss_spread_without_deterministic_mode(cuda):
    """Without the weight-gradient turnstile the FORWARD is still order independent (GroupNorm,
    split-K and the loss reduce in a fixed order): the loss of repeated runs is bit-identical; only
    the fp32 `red` accumulation of the LoRA gradients may differ in the last bits."""
    g, st = _make_step(cuda, 1)
    losses, grads = [], []
    for i in range(5):
        st.unet.lora_grad.zero_()
        st.forward_backward()
        torch.cuda.synchronize()
        losses.append(st.loss.item())
        grads.append(st.unet.lora_grad.clone())
    spread = (max(losses) - min(losses)) / abs(losses[0])
    gspread = max(_rel(x, grads[0]) for x in grads[1:])
    print(f"[determinism] loss spread over 5 runs {spread:.3e}; LoRA-gradient rel-L2 spread {gspread:.3e}", flush=True)
    assert spread == 0.0
    assert gspread <= 1e-5
