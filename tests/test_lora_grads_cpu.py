"""The per-tensor LoRA-gradient check of tests/grad_check.py on the CPU: the product's host plan (merged
student + teacher pass, tape, backward walk, flat gradient buffer) with every kernel replaced by its torch
semantics (tests/ops_interp.py), against float64 autograd and the bf16-emulating oracle.  CPU twin of
tests/test_lora_grads_gpu.py, so the checker itself - and its power to reject plausible plan bugs - is
tested on a machine without a GPU."""
import pytest
import torch

import grad_check
import ops_interp
from gemm_interp import build_net


def _sets(monkeypatch, cfg_name, B=2, hw=8, seed=5):
    from oracle import unet_ref
    from pcm_b200 import config
    ocfg, pcfg = getattr(unet_ref, cfg_name), getattr(config, cfg_name)
    P = unet_ref.init_params(ocfg, seed, lora_b_std=0.02)
    inp = grad_check.make_inputs(ocfg, B, hw, seed)
    ops_interp.install(monkeypatch)
    return grad_check.compute(f"{cfg_name} host plan, B={B}, {hw}x{hw}", ocfg, P,
                              lambda: build_net(pcfg, sd=P)[0], inp, "cpu")


@pytest.mark.parametrize("cfg_name", ["TINY", "TINY_XL"])
def test_host_plan_lora_grads_match_float64_per_tensor(monkeypatch, cfg_name):
    sets = _sets(monkeypatch, cfg_name)
    grad_check.assert_passes(grad_check.check(sets))
    grad_check.assert_mutations_rejected(sets)


def test_zero_reference_tensor_must_be_exactly_zero():
    ref = {"a": torch.zeros(4, 4, dtype=torch.float64), "b": torch.ones(4, 4, dtype=torch.float64)}
    sets = grad_check.GradSets("zero", {"a": torch.zeros(4, 4), "b": torch.ones(4, 4)}, dict(ref), ref)
    assert not grad_check.check(sets).failures
    tiny = {"a": torch.full((4, 4), 1e-30), "b": torch.ones(4, 4)}
    assert [r.key for r in grad_check.check(sets, tiny).failures] == ["a"]


def test_oracle_round_grads_only_changes_the_backward():
    """round_grads leaves the forward bit-identical and rounds only gradients: on the float32 oracle it
    moves the LoRA gradients by bf16-sized amounts, not more."""
    from oracle import unet_ref
    ocfg = unet_ref.TINY
    P = unet_ref.init_params(ocfg, 0)
    inp = grad_check.make_inputs(ocfg, 1, 8, 0)
    out = []
    for rg in (False, True):
        Pg = {k: (v.clone().requires_grad_(True) if ".lora_" in k else v) for k, v in P.items()}
        eps = unet_ref.UNetRef(ocfg, Pg, emulate_bf16=True, round_grads=rg)(inp["x"][:1], inp["ts"][:1], inp["ctx"][:1])
        (eps * inp["G"]).sum().backward()
        out.append((eps.detach(), {k: v.grad for k, v in Pg.items() if ".lora_" in k}))
    assert torch.equal(out[0][0], out[1][0])
    rel = [((out[1][1][k] - g).norm() / g.norm()).item() for k, g in out[0][1].items()]
    assert 0 < max(rel) < 0.1, max(rel)
