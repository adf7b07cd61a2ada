"""Gradient checkpointing (PCMTrainStep(gradient_checkpointing=True)) without a GPU.

Numbers: the product step runs on CPU with every kernel replaced by its torch semantics
(tests/ops_interp.py), once with the stored tape and once checkpointed, on the same weights and inputs.
The interpreter's CPU matmuls may block differently at B and 3B rows, so here the two agree to fp32
round-off; the bitwise claim is tests/test_checkpoint_gpu.py's.

Plan and memory: an SD1.5 bs 8, 64x64 step is dry-run (ops record instead of launching).  Every GEMM a
rebuilt block launches must carry the block_n / ksplit of the same launch in the merged pass, every rebuilt
GroupNorm the merged pass's partition batch, and the checkpointed tape must hold no merged-pass activation.

Data parallel: the 2-rank gloo step (as tests/test_dp_step_gloo.py) ends with the same parameters with
checkpointing on and off."""
import importlib.util
import os
import socket
import sys

import pytest
import torch

import ops_interp
from gemm_interp import BF16, refresh_operands

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def groupnorm_fwd_part(x1, x2, gamma, beta, eps, silu, out, stats, B, part_B, HW, G=32):
    """Torch semantics of ops.groupnorm_fwd_part: the partition batch only orders the kernel's sums."""
    assert part_B >= B
    return ops_interp.groupnorm_fwd(x1, x2, gamma, beta, eps, silu, out, stats, B, HW, G)


def _install(mp):
    from pcm_b200 import ops
    ops_interp.install_step(mp)
    mp.setattr(ops, "groupnorm_fwd_part", groupnorm_fwd_part)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _build(cfg, P, ckpt, **kw):
    from pcm_b200 import ops
    from pcm_b200.step import PCMTrainStep
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        st = PCMTrainStep(cfg, P, "cpu", gradient_checkpointing=ckpt, **kw)
    finally:
        ops.DRY_RUN = old
    refresh_operands(st.unet)
    return st


def _load(st, batch, xl):
    extra = dict(text_embeds=batch["text_embeds"].to(BF16), time_ids=batch["time_ids"]) if xl else {}
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF16), batch["uncond_prompt_embeds"].to(BF16), **extra)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


CASES = {
    "TINY": ("TINY", {}),
    "TINY_XL": ("TINY_XL", dict(num_ddim_timesteps=40)),
    "TINY_no_cfg_solver": ("TINY", dict(apply_cfg_solver=False)),
    "TINY_XL_no_cfg_solver": ("TINY_XL", dict(num_ddim_timesteps=40, apply_cfg_solver=False)),
    "TINY_ema": ("TINY", dict(ema_decay=0.95)),
    "TINY_two_substeps": ("TINY", dict(teacher_substeps=2)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_checkpointed_step_matches_the_stored_tape(monkeypatch, case):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    cfg_name, kw = CASES[case]
    xl = cfg_name == "TINY_XL"
    B, hw = 2, 8
    ocfg = getattr(unet_ref, cfg_name)
    P = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=0, **(dict(num_ddim=40, zero_uncond=True) if xl else {}))
    cfg = getattr(config, cfg_name)
    steps = [_build(cfg, P, ckpt, batch=B, height=hw, width=hw, multiphase=4, **kw)
             for ckpt in (False, True)]
    _install(monkeypatch)
    res = []
    p0 = steps[0].unet.lora_master.clone()
    for st in steps:
        _load(st, batch, xl)
        st.forward_backward()
        grad = st.unet.lora_grad.clone()
        st.optimizer_step()
        res.append(dict(loss=st.loss.clone(), grad=grad, master=st.unet.lora_master.clone(),
                        m=st.exp_avg.clone(), v=st.exp_avg_sq.clone()))
    ref, ck = res
    assert torch.equal(ck["loss"], ref["loss"])     # the forward is the same launches either way
    assert ref["grad"].abs().max() > 0 and ref["master"].ne(p0).any()
    for k in ("grad", "master", "m", "v"):
        assert _rel(ck[k], ref[k]) <= 1e-6, (k, _rel(ck[k], ref[k]))


# ---------------------------------------------------------------------------------------------
# dry run of the SD1.5 benchmark step: launch plans and tape
# ---------------------------------------------------------------------------------------------
def _step_memory():
    spec = importlib.util.spec_from_file_location("step_memory", os.path.join(ROOT, "tools", "step_memory.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def sd15_dry_run():
    """One checkpointed SD1.5 bs 8, 64x64 step, dry-run.  Returns the launch log (kernel records with their
    C-ABI arguments, and a ("block", kind, name, rebuilding, phase) marker around every block's forward)
    and the tape counts taken just before backward()."""
    from pcm_b200 import config, ops, weights
    from pcm_b200.step import PCMTrainStep
    from pcm_b200.unet import UNetB200
    sm = _step_memory()
    B, hw = 8, 64
    mp = pytest.MonkeyPatch()
    log = []
    try:
        mp.setattr(ops, "DRY_RUN", log)
        mp.setattr(ops, "_NUM_SMS", 132)
        mp.setattr(ops, "_call", lambda name, *args: log.append((name, args)))
        block = UNetB200._block

        def marked(self, kind, name, xs, P, save, up=False):
            log.append(("block", (kind, name, P.plan_b is not None, "begin")))
            r = block(self, kind, name, xs, P, save, up)
            log.append(("block", (kind, name, P.plan_b is not None, "end")))
            return r
        mp.setattr(UNetB200, "_block", marked)
        st = PCMTrainStep(config.SD15, weights.synthetic_state_dict(config.SD15, 0), "cpu", batch=B, height=hw,
                          width=hw, multiphase=4, gradient_checkpointing=True)
        tape = {}
        saved = {}
        bwd = st.unet.backward

        def counted(*a, **kw):
            s = st.unet.saved
            tape.update(sm.tape_bytes(s))
            saved["records"] = sm._tensors([s.tape, s.head], [])       # block records and the head GN
            saved["state"] = sm._tensors(s.rebuild, [])                # time embedding, context k / v
            saved["rows"] = s.shape[0]
            return bwd(*a, **kw)
        st.unet.backward = counted
        log.clear()
        st.run_eager()
    finally:
        mp.undo()
    return dict(log=log, tape=tape, saved=saved, B=B)


def _segments(log, rebuilding):
    """{block name: [launch records]} of the first forward (merged pass) or of the rebuilds."""
    segs, cur = {}, None
    for name, info in log:
        if name == "block":
            kind, bname, reb, edge = info
            if edge == "begin" and reb == rebuilding and bname not in segs:
                cur = segs.setdefault(bname, [])
                continue
            if edge == "end":
                cur = None
            continue
        if cur is not None:
            cur.append((name, info))
    return segs


def test_rebuilt_blocks_keep_the_merged_pass_launch_plan(sd15_dry_run):
    from pcm_b200 import ops
    log, B = sd15_dry_run["log"], sd15_dry_run["B"]
    merged, rebuilt = _segments(log, False), _segments(log, True)
    assert len(rebuilt) == len(merged) > 20
    replanned = gemms = gns = 0
    for name, seg in rebuilt.items():
        ref = merged[name]
        kinds = [k for k, _ in seg]
        assert [k.replace("_part", "") for k in kinds] == [k for k, _ in ref], name
        for (k, a), (_, r) in zip(seg, ref):
            if k == "gemm":
                gemms += 1
                assert (a["bn"], a["ksplit"], a["N"], a["K"], a["prog"]) == \
                    (r["bn"], r["ksplit"], r["N"], r["K"], r["prog"]), name
                assert a["M"] in (r["M"], r["M"] // 3), name       # main GEMMs: 3B -> B rows
                if ops.pick_tiling(a["M"], a["N"], a["K"] // 64) != (a["bn"], a["ksplit"]):
                    replanned += 1      # the rebuild's own M would have picked another tiling
            elif k == "pcm_groupnorm_fwd_part":
                gns += 1
                # (x1, x2, C1, C2, B, part_B, HW, ...) against the merged (x1, x2, C1, C2, B, HW, ...)
                assert a[4] == B and a[5] == r[4] == 3 * B and a[6] == r[5] and a[2:4] == r[2:4], name
        assert "pcm_groupnorm_fwd" not in kinds, name
    assert gemms > 100 and gns > 40
    assert replanned > 0


def test_checkpointed_tape_keeps_only_student_rows(sd15_dry_run):
    """SD1.5 bs 8, 64x64: the stored tape keeps about 17 GiB alive (tools/step_memory.py --dry-run); the
    checkpointed one less than 1 GiB, with no storage of a 3B-row activation reachable."""
    tape, saved, B = sd15_dry_run["tape"], sd15_dry_run["saved"], sd15_dry_run["B"]
    assert saved["rows"] == B
    assert tape["tape_gib"] < 1.0 and 0.4 < tape["block_inputs_gib"] < 0.6, tape
    assert tape["row_view_gib"] < 0.15, tape        # only the pass's time-embedding / context projections
    # every tensor of the records is an owned copy of student rows (block inputs: NHWC, B samples)
    for t in saved["records"]:
        assert t.untyped_storage().nbytes() == t.numel() * t.element_size(), tuple(t.shape)
        assert t.shape[0] == (B if t.dim() == 4 else B * 64 * 64 if t.dim() == 2 else B), tuple(t.shape)
    # the per-pass state: student-row views of the time-embedding and context projections (3B rows of a
    # few small matrices) and of the step's context input
    state = {t.untyped_storage().data_ptr(): t.untyped_storage().nbytes() for t in saved["state"]}
    assert sum(state.values()) < 0.15 * (1 << 30), sum(state.values())


# ---------------------------------------------------------------------------------------------
# data parallel (gloo, 2 ranks)
# ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    here = os.path.dirname(os.path.abspath(__file__))
    for p in (here, os.path.dirname(here)):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      PCM_DP_OVERLAP="1")
    torch.set_num_threads(2)
    import torch.distributed as dist
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, dp

    class MP:
        @staticmethod
        def setattr(obj, name, val):
            setattr(obj, name, val)

    pg = dp.init_process_group("gloo")
    B, hw = 2, 8
    P = unet_ref.init_params(unet_ref.TINY, 0, lora_b_std=0.02)
    batch = pcm_ref.make_batch(unet_ref.TINY, B, hw, seed=dp.rank_seed(11, rank))
    kw = dict(batch=B, height=hw, width=hw, multiphase=4, weight_decay=1e-2, max_grad_norm=1.0,
              process_group=pg)
    steps = [_build(config.TINY, P, ckpt, **kw) for ckpt in (False, True)]
    _install(MP)
    masters, p0 = [], steps[0].unet.lora_master.clone()
    for st in steps:
        assert len(st.reducer.buckets) > 1
        _load(st, batch, False)
        st.step()
        masters.append(st.unet.lora_master.clone())
    if rank == 0:
        out["rel"] = _rel(masters[1], masters[0])
        out["moved"] = (masters[0] - p0).abs().max().item()
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_checkpointed_step_matches_the_stored_tape():
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    assert out["moved"] > 0 and out["rel"] <= 1e-6, dict(out)
