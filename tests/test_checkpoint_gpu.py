"""Gradient checkpointing on the GPU: PCMTrainStep(gradient_checkpointing=True) computes bit for bit what
the stored-tape step computes (the rebuilt blocks keep the merged pass's GEMM tiling and GroupNorm
partition), keeps far less memory alive, and runs the SDXL 1024x1024 step that does not fit without it."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
GIB = float(1 << 30)


def _inputs(cfg, B, hw, seed=100):
    g = torch.Generator().manual_seed(seed)
    t = dict(latents=torch.randn(B, hw, hw, 4, generator=g), noise=torch.randn(B, hw, hw, 4, generator=g),
             index=torch.randint(0, 40 if cfg.addition_embed else 50, (B,), generator=g),
             w=4.0 + torch.rand(B, generator=g),
             prompt=torch.randn(B, 77, cfg.cross_attention_dim, generator=g).to(BF),
             uncond=torch.randn(B, 77, cfg.cross_attention_dim, generator=g).to(BF))
    if cfg.addition_embed:
        t["uncond"].zero_()
        t["text_embeds"] = torch.randn(B, cfg.text_embed_dim, generator=g).to(BF)
        t["time_ids"] = torch.tensor([[hw * 8, hw * 8, 0, 0, hw * 8, hw * 8]] * B)
    return t


def _load(st, t):
    st.load_inputs(t["latents"], t["noise"], t["index"], t["w"], t["prompt"], t["uncond"],
                   text_embeds=t.get("text_embeds"), time_ids=t.get("time_ids"))


def _step(cfg, sd, dev, B, hw, ckpt, **kw):
    from pcm_b200.step import PCMTrainStep
    return PCMTrainStep(cfg, sd, dev, batch=B, height=hw, width=hw, multiphase=4,
                        num_ddim_timesteps=40 if cfg.addition_embed else 50, lr=5e-6, weight_decay=1e-3,
                        max_grad_norm=1.0, gradient_checkpointing=ckpt, **kw)


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _run_both_ways(cfg, sd, dev, B, hw):
    """{mode: {eager / graph results}} for the stored-tape and the checkpointed step on the same inputs."""
    inp = _inputs(cfg, B, hw)
    out = {}
    for ckpt in (False, True):
        st = _step(cfg, sd, dev, B, hw, ckpt)
        _load(st, inp)
        st.forward_backward()
        res = dict(loss=st.loss.clone(), grad=st.unet.lora_grad.clone())
        st.optimizer_step()
        res.update(master=st.unet.lora_master.clone(), m=st.exp_avg.clone(), v=st.exp_avg_sq.clone())
        st.capture(warmup=1)            # restores the state after the eager step when it is done
        for _ in range(2):
            st.step()
        torch.cuda.synchronize()
        res.update(g_loss=st.loss.clone(), g_master=st.unet.lora_master.clone(), g_m=st.exp_avg.clone(),
                   g_v=st.exp_avg_sq.clone())
        out[ckpt] = {k: v.cpu() for k, v in res.items()}
        st.graph = None
        del st
        _free()
    return out


@pytest.fixture
def deterministic(cuda):
    from pcm_b200 import ops
    ops.deterministic(True, cuda)
    yield
    ops.deterministic(False)


def _bitwise(out):
    a, b = out[False], out[True]
    for k in a:
        assert torch.equal(a[k], b[k]), (k, (a[k] - b[k]).abs().max().item())
    assert a["grad"].abs().max() > 0 and torch.isfinite(a["loss"]).all()


@pytest.mark.parametrize("cfg_name,B,hw", [("SD15", 8, 64), ("TINY_XL", 2, 16)])
def test_checkpointed_step_is_bitwise_the_stored_tape_step(cuda, deterministic, cfg_name, B, hw):
    """Loss, lora_grad and the updated lora_master / exp_avg / exp_avg_sq after one eager step, then loss and
    optimiser state after two more steps replayed from a CUDA graph, with and without checkpointing."""
    from pcm_b200 import config, weights
    cfg = getattr(config, cfg_name)
    sd = weights.synthetic_state_dict(cfg, 0)
    _bitwise(_run_both_ways(cfg, sd, cuda, B, hw))


def _peak(cfg, sd, dev, B, hw, ckpt):
    torch.zeros(1, device=dev)     # the allocator of a fresh process exists after its first allocation
    _free()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    st = _step(cfg, sd, dev, B, hw, ckpt)
    _load(st, _inputs(cfg, B, hw))
    st.run_eager()
    st.run_eager()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - base
    del st
    _free()
    return peak


def test_checkpointing_halves_the_sd15_step_memory(cuda):
    """SD1.5 bs 8, 64x64, eager steps.  The dry run (tools/step_memory.py --dry-run) counts 17.35 GiB of tape
    storage without checkpointing and 0.54 GiB with it; the peak must drop by at least half of the
    difference.  Measured on an H100 80GB HBM3 (400 W power limit): peak allocated 25.85 GiB with the
    stored tape, 6.26 GiB checkpointed (a drop of 19.6 GiB: the tape, and the merged pass's activations
    that the forward no longer keeps)."""
    from pcm_b200 import config, weights
    cfg = config.SD15
    sd = weights.synthetic_state_dict(cfg, 0)
    off = _peak(cfg, sd, cuda, 8, 64, False)
    on = _peak(cfg, sd, cuda, 8, 64, True)
    print(f"[sd15 bs 8] peak allocated: stored tape {off / GIB:.2f} GiB, checkpointed {on / GIB:.2f} GiB")
    assert off - on >= PEAK_DROP_GIB * GIB, (off / GIB, on / GIB)


PEAK_DROP_GIB = 8.4         # half of the 16.8 GiB the dry run predicts the checkpointed tape saves


def test_sdxl_1024_bs4_checkpointed_step_runs_under_graph_capture(cuda):
    """BASELINE config 4 (SDXL, 1024x1024 -> 128x128 latents, bs 4 per GPU), synthetic weights: the
    checkpointed step captures and replays with a finite loss.  Measured on an H100 80GB HBM3 (400 W power
    limit): 20.6 GiB peak allocated; the stored-tape step runs out of memory (tools/step_memory.py)."""
    from pcm_b200 import config, weights
    cfg = config.SDXL
    B, hw = 4, 128
    st = _step(cfg, weights.synthetic_state_dict(cfg, 0), cuda, B, hw, True)
    _free()
    _load(st, _inputs(cfg, B, hw))
    st.capture(warmup=1)
    st.step()
    torch.cuda.synchronize()
    print(f"[sdxl 1024 bs 4, checkpointed] loss {st.loss.item():.6f}, peak allocated "
          f"{torch.cuda.max_memory_allocated(cuda) / GIB:.2f} GiB")
    assert torch.isfinite(st.loss).all() and st.opt_state[1].item() == 1.0
    st.graph = None
    del st
    _free()


def test_entry_point_gradient_checkpointing_is_bitwise(cuda, tmp_path):
    """train_pcm_lora_sd15.main() with --gradient_checkpointing: 2 steps, the checkpoint it writes equals the
    one of the same run without the flag, bit for bit."""
    from pcm_b200 import config, ops, train_pcm_lora_sd15 as T
    ops.deterministic(True, cuda)
    try:
        states = []
        for flag in ([], ["--gradient_checkpointing"]):
            out = tmp_path / ("ckpt" if flag else "plain")
            a = T.parse_args(["--synthetic", "--output_dir", str(out), "--train_batch_size", "2", "--resolution",
                              "128", "--multiphase", "4", "--seed", "5", "--mixed_precision", "bf16",
                              "--learning_rate", "1e-3", "--max_train_steps", "2", "--checkpointing_steps", "2",
                              "--log_every", "1", "--w_min", "4", "--w_max", "5"] + flag)
            a._cfg = config.TINY
            st = T.main(a)
            assert st.unet.gradient_checkpointing == bool(flag)
            states.append(torch.load(out / "checkpoint-2" / "pcm_b200_state.pt"))
            del st
            _free()
        plain, ck = states
        for k in ("lora_master", "exp_avg", "exp_avg_sq", "opt_state"):
            assert torch.equal(plain[k], ck[k]), k
        assert plain["opt_state"][1].item() == 2.0
    finally:
        ops.deterministic(False)
