"""Data-parallel plumbing of the step (one process per GPU, torch.distributed).

The reference wraps the student in DistributedDataParallel through accelerate
(train_pcm_lora_sd15.py:1034): bucketed all-reduce(mean) of the LoRA gradients overlapped with the
backward pass, `set_seed(args.seed + process_index)` (:795-797), then clip_grad_norm_ on the
reduced gradient (:1297-1298).  Here the LoRA gradients live in ONE flat fp32 buffer laid out in
forward order, so the backward pass completes it from the END: `GradReducer` cuts the buffer into
a few contiguous buckets on block boundaries and launches `all_reduce(SUM)` of a bucket (async, on
NCCL's own stream, ordered after the weight-gradient stream) as soon as the backward has passed the
bucket's first layer - the exchange overlaps the rest of the backward like DDP's.  The 1/world
average and the clip coefficient are folded into the AdamW kernel (`pcm_adamw_clip`), which
therefore needs the sum of squares of the SUMMED gradient.
"""
import math
import os

import torch.distributed as dist


def env_rank_world():
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def rank_seed(base_seed, rank):
    """accelerate.utils.set_seed(args.seed + accelerator.process_index)."""
    return int(base_seed) + int(rank)


def init_process_group(backend="nccl", device=None):
    """NVLink-only NCCL defaults for one 8-GPU NVSwitch box (8xH100 SXM); rendezvous from MASTER_* env."""
    if backend == "nccl":
        os.environ.setdefault("NCCL_IB_DISABLE", "1")
        os.environ.setdefault("NCCL_P2P_LEVEL", "NVL")
        os.environ.setdefault("NCCL_NVLS_ENABLE", "1")
        dist.init_process_group("nccl", device_id=device)
    else:
        dist.init_process_group(backend)
    return dist.group.WORLD


def allreduce_flat_grad(flat_grad, group=None):
    """One collective: SUM over ranks of the flat LoRA gradient (269 MB fp32 for SD1.5 r=64)."""
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return flat_grad


def bucket_bounds(block_offsets, total, num_buckets):
    """Cut [0, total) into <= num_buckets contiguous ranges of similar size whose boundaries are
    block starts (`block_offsets`: ascending first-element offsets of the UNet blocks that own LoRA
    layers).  Returned ascending; the LAST range is the first one the backward pass completes."""
    offs = sorted(set(int(o) for o in block_offsets if 0 < o < total))
    cuts = []
    for k in range(1, max(1, num_buckets)):
        want = total * k // num_buckets
        if not offs:
            break
        best = min(offs, key=lambda o: abs(o - want))
        if best not in cuts:
            cuts.append(best)
    edges = [0] + sorted(cuts) + [total]
    return [(edges[i], edges[i + 1]) for i in range(len(edges) - 1) if edges[i + 1] > edges[i]]


class GradReducer:
    """Bucketed, backward-overlapped SUM all-reduce of the flat LoRA gradient.

    ready(lo): every gradient element at offset >= lo is final (the backward pass just finished the
    block whose first LoRA layer starts at `lo`); call it on the stream that wrote the gradients.
    finish(): make the current stream wait for all launched collectives (and launch the rest)."""

    def __init__(self, flat_grad, block_offsets, group=None, num_buckets=4):
        self.grad, self.group = flat_grad, group
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        self.buckets = bucket_bounds(block_offsets, flat_grad.numel(), num_buckets)
        self._next = len(self.buckets) - 1
        self._work = []

    def start(self):
        self._next = len(self.buckets) - 1
        self._work = []

    def ready(self, lo):
        if self.world == 1:
            return
        while self._next >= 0 and self.buckets[self._next][0] >= lo:
            a, b = self.buckets[self._next]
            self._work.append(dist.all_reduce(self.grad[a:b], op=dist.ReduceOp.SUM, group=self.group,
                                              async_op=True))
            self._next -= 1

    def finish(self):
        self.ready(0)
        for w in self._work:
            w.wait()          # current stream waits for the collective's stream (no host block)
        self._work = []


def folded_coef(sumsq_of_sum, world, max_norm):
    """Scalar applied to the SUMMED gradient so that it equals clip(mean-gradient):
    norm(mean) = sqrt(sumsq)/world ; coef = min(1, max_norm/(norm+1e-6)) / world.
    Mirrors adamw_clip_kernel (csrc/optim.cu); used for logging and by the gloo tests."""
    norm = math.sqrt(float(sumsq_of_sum)) / world
    c = min(max_norm / (norm + 1e-6), 1.0) if max_norm > 0 else 1.0
    return c / world, norm
