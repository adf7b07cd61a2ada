"""2-rank NCCL test of the PRODUCT data-parallel path (PCMTrainStep with a process group: bucketed
all-reduce(SUM) overlapped with the backward pass, 1/world and the clip folded into pcm_adamw_clip):
two ranks with DIFFERENT batches must end with bit-identical LoRA parameters, equal to a single
process applying clip_grad_norm_ + AdamW to the MEAN of the two local gradients - what DDP +
accelerate do in the reference (train_pcm_lora_sd15.py:1034, 1296-1301).  Needs 2 GPUs
(`python -m pytest tests/test_dp_nccl_gpu.py -m gpu` on a 2-GPU machine); skipped otherwise."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _worker(rank, world, port, out, use_graph):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, dp, ops
    from pcm_b200.step import PCMTrainStep
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    pg = dp.init_process_group("nccl", dev)
    ops.deterministic(True, dev)
    B, hw, mp = 2, 16, 4
    P = unet_ref.init_params(unet_ref.TINY, 0)                       # replicated weights
    batch = pcm_ref.make_batch(unet_ref.TINY, B, hw, seed=dp.rank_seed(11, rank))   # per-rank data
    args = (_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
            batch["prompt_embeds"].to(BF), batch["uncond_prompt_embeds"].to(BF))
    kw = dict(batch=B, height=hw, width=hw, multiphase=mp, lr=1e-3, weight_decay=1e-2, max_grad_norm=1.0)
    # local gradient of this rank (single-process object, no collective)
    solo = PCMTrainStep(config.TINY, P, dev, **kw)
    solo.load_inputs(*args)
    solo.forward_backward()
    torch.cuda.synchronize()
    g_local = solo.unet.lora_grad.clone()
    names = solo.unet.lora_grad_dict()
    # the product data-parallel step
    st = PCMTrainStep(config.TINY, P, dev, process_group=pg, **kw)
    assert len(st.reducer.buckets) > 1
    st.load_inputs(*args)
    if use_graph:
        st.capture(warmup=1)
    st.step()
    torch.cuda.synchronize()
    gathered = [torch.zeros_like(g_local) for _ in range(world)]
    dist.all_gather(gathered, g_local)
    master = st.unet.lora_master.clone()
    masters = [torch.zeros_like(master) for _ in range(world)]
    dist.all_gather(masters, master)
    if rank == 0:
        out["masters_equal"] = all(torch.equal(masters[0], m) for m in masters[1:])
        # expected: mean gradient -> clip_grad_norm_(1.0) -> AdamW (oracle restatement, CPU)
        mean = (sum(g.double() for g in gathered) / world).float().cpu()
        params = {"w": solo.unet.lora_master.detach().cpu().clone()}     # = initial parameters
        pcm_ref.clip_and_adamw_ref(params, {"w": mean}, {}, lr=1e-3, weight_decay=1e-2, max_grad_norm=1.0)
        out["max_abs_err"] = (master.cpu() - params["w"]).abs().max().item()
        out["update_size"] = (params["w"] - solo.unet.lora_master.cpu()).abs().max().item()
        out["num_lora"] = len(names)
    dist.barrier()
    st.graph = st.graph_opt = None
    torch.cuda.synchronize()
    dist.destroy_process_group()


@pytest.mark.parametrize("use_graph", [False, True])
def test_two_rank_update_matches_mean_gradient_adamw(use_graph):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out, use_graph), nprocs=world, join=True)
    assert out["masters_equal"], "ranks ended with different parameters"
    assert out["update_size"] > 1e-5                      # the step really moved the parameters
    assert out["max_abs_err"] <= 1e-6 + 1e-3 * out["update_size"], dict(out)
