"""Every LoRA gradient of the full-width UNet backward, tensor by tensor, against float64 autograd.

Each configuration runs the merged pass every training step runs - forward(3B rows, lora_batch=B,
save=True), the teacher rows with inputs of their own - then backward(G) of the student rows, and holds
each of the LoRA tensors, the student rows of eps and the teacher rows of eps to the rule of
tests/grad_check.py: at most twice the error of the bf16-emulating oracle, measured against float64.
The last test runs the whole PCM step with the L2 loss against the oracle's step in float64.

One reference network lives on the device at a time and is freed before the next; each test prints its
tensor count, the prod / base error ratios, the worst tensor, its device-memory peak and its wall time.
"""
import dataclasses
import time

import pytest
import torch

import grad_check

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _sets(cuda, cfg_name, *, B, hw, rank=64, lora_b_std=0.02, seed=0):
    from oracle import unet_ref
    from pcm_b200 import config
    from pcm_b200.unet import UNetB200
    ocfg = dataclasses.replace(getattr(unet_ref, cfg_name), lora_rank=rank)
    pcfg = dataclasses.replace(getattr(config, cfg_name), lora_rank=rank)
    P = unet_ref.init_params(ocfg, seed, lora_b_std=lora_b_std)
    inp = grad_check.make_inputs(ocfg, B, hw, seed)
    name = f"{cfg_name} rank {rank}, B={B}, {hw}x{hw}" + (", B=0 init" if lora_b_std == 0 else "")
    return grad_check.compute(name, ocfg, P, lambda: UNetB200(pcfg, P, cuda), inp, cuda)


def test_sd15_merged_pass_lora_grads(cuda):
    sets = _sets(cuda, "SD15", B=2, hw=32)
    grad_check.assert_passes(grad_check.check(sets))
    grad_check.assert_mutations_rejected(sets)


def test_sd15_benchmark_latents_lora_grads(cuda):
    """64 x 64 latents: 4096-token self-attention, the benchmark's latent size."""
    grad_check.assert_passes(grad_check.check(_sets(cuda, "SD15", B=1, hw=64)))


@pytest.mark.parametrize("rank", [8, 256])
def test_sd15_lora_grads_at_rank(cuda, rank):
    """Rank 8: one K block narrower than 64 and weight-gradient slices ending inside stacked T / dT columns;
    rank 256: four 64-wide K chunks and rank slices."""
    grad_check.assert_passes(grad_check.check(_sets(cuda, "SD15", B=2, hw=32, rank=rank)))


def test_sd15_peft_initialisation_lora_grads(cuda):
    """B = 0 (peft's initialisation): dT = s B^T dy vanishes, so every A-gradient is exactly zero."""
    sets = _sets(cuda, "SD15", B=2, hw=32, lora_b_std=0.0)
    a = [k for k in sets.ref if k.endswith("lora_A.weight")]
    assert a and all(sets.ref[k].abs().max().item() == 0 for k in a)
    assert all(sets.prod[k].abs().max().item() == 0 for k in a), [k for k in a if sets.prod[k].abs().max() > 0][:4]
    grad_check.assert_passes(grad_check.check(sets))


def test_sdxl_merged_pass_lora_grads(cuda):
    """SDXL at full width with added conditions: 60 cross-attention layers at 1280 in context chunks."""
    sets = _sets(cuda, "SDXL", B=1, hw=32)
    grad_check.assert_passes(grad_check.check(sets))
    grad_check.assert_mutations_rejected(sets)


def test_l2_step_lora_grads(cuda):
    """PCMTrainStep(loss_type="l2").forward_backward() at SD1.5 width (bs 1, 32 x 32 latents, 2 phases)
    against pcm_step_ref in float64: the loss seed, the teacher step and the target pass feeding the
    backward.  The L2 gradient is linear in model_pred - target, so unlike Huber's ~sign(d) it does not
    turn bf16 noise in d into gradient noise."""
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    from pcm_b200.step import PCMTrainStep
    ocfg = unet_ref.SD15
    P = unet_ref.init_params(ocfg, 0)
    batch = pcm_ref.make_batch(ocfg, 1, 32, seed=0)
    for k in ("prompt_embeds", "uncond_prompt_embeds"):      # the step takes bf16 embeddings
        batch[k] = grad_check.bf16_exact(batch[k])
    grad_check.reset_peak(cuda)
    t0 = time.perf_counter()
    nhwc = grad_check._nhwc
    st = PCMTrainStep(config.SD15, P, cuda, batch=1, height=32, width=32, multiphase=2, loss_type="l2")
    st.load_inputs(nhwc(batch["latents"]), nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF16), batch["uncond_prompt_embeds"].to(BF16))
    st.forward_backward()
    torch.cuda.synchronize()
    prod = st.unet.lora_grad_dict()
    del st
    torch.cuda.empty_cache()

    def on(dtype):
        return {k: (v.to(cuda, dtype) if v.is_floating_point() else v.to(cuda)) for k, v in batch.items()}

    kw = dict(multiphase=2, loss_type="l2", need_grad=True)
    with grad_check.full_fp32():
        ref = pcm_ref.pcm_step_ref(ocfg, grad_check.ref_params(P, torch.float64, cuda), on(torch.float64),
                                   emulate_bf16=False, round_inputs=True, **kw)["grads"]
        torch.cuda.empty_cache()
        base = pcm_ref.pcm_step_ref(ocfg, {k: v.to(cuda) for k, v in P.items()}, on(torch.float32),
                                    emulate_bf16=True, round_grads=True, **kw)["grads"]
    torch.cuda.synchronize()
    sets = grad_check.GradSets("SD15 L2 step, bs 1, 32x32, 2 phases", prod, base, ref,
                               peak_gib=torch.cuda.max_memory_allocated(cuda) / 2 ** 30,
                               wall_s=time.perf_counter() - t0)
    grad_check.assert_passes(grad_check.check(sets))
