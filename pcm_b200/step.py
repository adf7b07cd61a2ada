"""One PCM-LoRA distillation iteration on the CUDA path: the body of the reference loop
train_pcm_lora_sd15.py:1139-1301 (noise / phase bookkeeping, student forward, teacher CFG DDIM
step, target forward, Huber loss, backward, gradient all-reduce, clip + AdamW) as a fixed sequence
of C-ABI kernel launches, capturable in ONE CUDA graph (no host sync inside; `index`, `w`,
timesteps, lr and the optimiser step counter live in device memory).
"""
import os

import numpy as np
import torch

from . import dp, ops
from .config import UNetConfig
from .unet import UNetB200

BF16 = torch.bfloat16


def sd15_alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012):
    """`scaled_linear` betas of the SD1.5 DDPMScheduler config (scheduling_ddpm_modified.py:211-215)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def inference_indices(num_ddim, multiphase):
    """Phase start indices, np.floor(np.linspace(0, N, multiphase, endpoint=False))
    (train_pcm_lora_sd15.py:1157-1160 / :322-325)."""
    return np.floor(np.linspace(0, num_ddim, num=multiphase, endpoint=False)).astype(np.int64)


class PCMTrainStep:
    """State + one-iteration driver.  All tensors NHWC; latents fp32 [B, H, W, 4]."""

    def __init__(self, cfg: UNetConfig, state_dict, device, *, batch, height, width, multiphase=4,
                 num_ddim_timesteps=50, num_train_timesteps=1000, loss_type="huber", huber_c=1e-3,
                 lr=5e-6, betas=(0.9, 0.999), adam_eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0,
                 apply_cfg_solver=True, bf16_mode=True, alphas_cumprod=None, process_group=None,
                 keep_debug=False, prediction_type="epsilon", ema_decay=None, grad_buckets=4,
                 teacher_substeps=1, gradient_checkpointing=False):
        """prediction_type: "epsilon" | "v_prediction" (predicted_origin, T15:268-280).
        ema_decay: None (reference behaviour: the target network IS the student, update_ema is never
        called, T15:1261-1268) or a rate in (0, 1): opt-in EMA target, updated after every optimiser
        step as update_ema does (T15:344-355).
        teacher_substeps: 1 (reference behaviour: ONE DDIM step of the teacher over the 20-timestep
        interval, T15:1217-1258) or k > 1 dividing the interval: the teacher is evaluated k times along
        it (opt-in multi-substep solve; each extra sub-step costs two more teacher forwards).
        gradient_checkpointing: the merged pass keeps only the student rows of each UNet block's inputs and
        the backward runs every block's student forward again right before its backward (diffusers'
        per-block torch.utils.checkpoint): less memory, one more student forward per step, the same
        numbers bit for bit."""
        ratio = num_train_timesteps // num_ddim_timesteps
        if teacher_substeps < 1 or ratio % teacher_substeps != 0:
            raise ValueError(f"teacher_substeps must divide the DDIM interval ({ratio} train timesteps)")
        self.substeps, self.sub_dt = teacher_substeps, ratio // teacher_substeps
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"Prediction type {prediction_type} currently not supported.")  # T15:277-278
        self.pred_type = 0 if prediction_type == "epsilon" else 1
        self.cfg, self.dev = cfg, device
        self.B, self.H, self.W = batch, height, width
        self.per = height * width * 4
        self.unet = UNetB200(cfg, state_dict, device, need_backward=True, lora=True,
                             gradient_checkpointing=gradient_checkpointing)
        self.multiphase, self.num_ddim, self.num_train = multiphase, num_ddim_timesteps, num_train_timesteps
        self.loss_type = 0 if loss_type == "huber" else 1
        self.huber_c = huber_c
        self.betas, self.adam_eps, self.wd, self.max_norm = betas, adam_eps, weight_decay, max_grad_norm
        self.apply_cfg = apply_cfg_solver
        self.bf16_mode = int(bf16_mode)
        self.pg = process_group
        self.world = 1 if process_group is None else torch.distributed.get_world_size(process_group)
        self.reducer = dp.GradReducer(self.unet.lora_grad, self.unet.block_grad_offsets().values(),
                                      group=process_group, num_buckets=grad_buckets) if self.world > 1 else None
        self.ema_decay = ema_decay
        self.ema_master = self.unet.lora_master.clone() if ema_decay is not None else None
        acp = sd15_alphas_cumprod(num_train_timesteps) if alphas_cumprod is None else alphas_cumprod
        self.acp = acp.float().to(device)
        self.inf_idx = torch.from_numpy(inference_indices(num_ddim_timesteps, multiphase)).to(device)
        f32 = dict(device=device, dtype=torch.float32)
        i64 = dict(device=device, dtype=torch.int64)
        B = batch
        self.coef = torch.zeros(B, 16, device=device, dtype=torch.float64)
        self.start_t, self.t, self.end_t = (torch.zeros(B, **i64) for _ in range(3))
        self.x_prev = torch.zeros(B, height, width, 4, **f32)
        self.d_eps = torch.zeros_like(self.x_prev)
        self.loss = torch.zeros(1, **f32)
        self.model_pred = torch.zeros_like(self.x_prev) if keep_debug else None
        self.target = torch.zeros_like(self.x_prev) if keep_debug else None
        n = self.unet.lora_master.numel()
        self.exp_avg = torch.zeros(n, **f32)
        self.exp_avg_sq = torch.zeros(n, **f32)
        self.opt_state = torch.tensor([lr, 0.0], **f32)  # lr, step
        # [0] = sum of squares; rest = scratch of the fixed-order reduction (PCM_SUMSQ_WS_DOUBLES)
        self.sumsq = torch.zeros(1024, device=device, dtype=torch.float64)
        self.debug = {} if keep_debug else None
        # static input slots (graph replay copies into these)
        self.in_latents = torch.zeros(B, height, width, 4, **f32)
        self.in_noise = torch.zeros_like(self.in_latents)
        self.in_index = torch.zeros(B, **i64)
        self.in_w = torch.zeros(B, **f32)
        # prompt and uncond embeddings are the two halves of ONE buffer so that the two teacher
        # passes of the CFG solve (T15:1219-1244) run as a single batch-2B forward
        # student + teacher(cond) + teacher(uncond) run as ONE batch-3B pass (LoRA on the first B
        # samples only): ctx3 = [prompt; prompt; uncond], noisy3 = 3 x noisy
        self.in_ctx3 = torch.zeros(3 * B * 77, cfg.cross_attention_dim, device=device, dtype=BF16)
        self.in_prompt = self.in_ctx3[:B * 77]
        self.in_uncond = self.in_ctx3[2 * B * 77:]
        self.noisy3 = torch.zeros(3 * B, height, width, 4, **f32)
        self.noisy = self.noisy3[:B]
        self.start_t3 = torch.zeros(3 * B, **i64)
        # SDXL added_cond_kwargs (train_pcm_lora_sdxl_adv.py:1094-1133): pooled text embedding + time ids,
        # laid out like ctx3 = [prompt; prompt; uncond]; the unconditional rows keep ZERO text embeddings
        # (uncond_pooled_prompt_embeds, :1215-1221) and the same time ids
        self.addc = cfg.addition_embed
        if self.addc:
            self.in_text3 = torch.zeros(3 * B, cfg.text_embed_dim, device=device, dtype=BF16)
            self.in_time_ids3 = torch.zeros(3 * B, cfg.num_time_ids, **i64)
        # data parallel: overlap the gradient all-reduce with the backward pass (PCM_DP_OVERLAP=0: one
        # flat all-reduce after the backward)
        self._overlap = os.environ.get("PCM_DP_OVERLAP", "1") != "0"
        self.graph = None
        self.graph_opt = None

    def set_lr(self, lr):
        self.opt_state[0] = lr

    # -- the iteration ------------------------------------------------------------------
    def forward_backward(self):
        """Everything up to (and including) the LoRA gradients, from the static input slots."""
        u, B, per = self.unet, self.B, self.per
        ops._call("pcm_prepare", self.acp.data_ptr(), self.num_train, self.num_ddim, self.inf_idx.data_ptr(),
                  self.multiphase, self.in_index.data_ptr(), self.in_w.data_ptr(), B, self.bf16_mode,
                  self.coef.data_ptr(), self.start_t.data_ptr(), self.t.data_ptr(), self.end_t.data_ptr())
        ops._call("pcm_add_noise", self.in_latents.data_ptr(), self.in_noise.data_ptr(), self.coef.data_ptr(),
                  per, B, self.bf16_mode, self.noisy.data_ptr())
        nb = 3 if self.apply_cfg else 2
        for i in range(1, nb):   # replicate the noisy latents for the teacher samples
            ops._call("pcm_add_noise", self.in_latents.data_ptr(), self.in_noise.data_ptr(),
                      self.coef.data_ptr(), per, B, self.bf16_mode, self.noisy3[i * B:(i + 1) * B].data_ptr())
            self.start_t3[i * B:(i + 1) * B].copy_(self.start_t)
        self.start_t3[:B].copy_(self.start_t)
        self.in_ctx3[B * 77:2 * B * 77].copy_(self.in_prompt)

        def added(lo, hi):
            return (self.in_text3[lo:hi], self.in_time_ids3[lo:hi]) if self.addc else None
        # one pass: [student | teacher cond | teacher uncond]; LoRA only on the student samples
        eps_all = u.forward(self.noisy3[:nb * B], self.start_t3[:nb * B],
                            self.in_ctx3 if nb == 3 else self.in_ctx3[:2 * B * 77],
                            lora=True, save=True, lora_batch=B, added_cond=added(0, nb * B))
        kv = u.saved_ctx_kv()
        eps_s, eps_c = eps_all[:B], eps_all[B:2 * B]
        eps_u = eps_all[2 * B:] if nb == 3 else eps_c
        # the target network is the student (same LoRA factors) on the same prompt embeddings
        # (T15:1192-1198 vs 1263-1268): its cross-attention k / v ARE the student rows of the pass above
        if kv is not None:
            kv = u.ctx_kv_rows(kv, self.in_prompt.shape[0]) if self.ema_master is None else None
        if self.substeps == 1:
            self.teacher_step_kernel(eps_c, eps_u)
        else:
            self._teacher_substeps(eps_c, eps_u, added)
        if self.ema_master is not None:      # opt-in EMA target: same network, EMA LoRA factors
            u.refresh_lora(self.ema_master)
        eps_t = u.forward(self.x_prev, self.t, self.in_prompt, lora=True, added_cond=added(0, B), ctx_kv=kv)
        if self.ema_master is not None:
            u.refresh_lora()
        self.loss_kernel(eps_s, eps_t)
        if self.debug is not None:
            self.debug.update(eps_student=eps_s, eps_cond=eps_c, eps_uncond=eps_u, eps_target=eps_t)
        if self.reducer is not None and self._overlap:
            # data parallel: bucketed all-reduce(SUM) launched from inside the backward pass
            self.reducer.start()
            u.backward(self.d_eps, grad_ready=self.reducer.ready)
            self.reducer.finish()
        else:
            u.backward(self.d_eps)

    def _teacher_substeps(self, eps_c, eps_u, added):
        """k DDIM sub-steps from start_t down to start_t - ratio (= t): the first uses the merged pass's
        teacher outputs, each further one runs the frozen teacher (cond + uncond, batch 2B) again."""
        u, B, k = self.unet, self.B, self.substeps
        x_cur = self.noisy
        t_cur = self.start_t
        nb = 2 if self.apply_cfg else 1
        for j in range(k):
            t_next = self.start_t - (j + 1) * self.sub_dt          # -1 for index 0: the solver's acp[0] entry
            out = self.x_prev if j == k - 1 else torch.empty_like(self.x_prev)
            ops._call("pcm_teacher_substep", eps_c.data_ptr(), eps_u.data_ptr(), x_cur.data_ptr(),
                      self.acp.data_ptr(), t_cur.data_ptr(), t_next.data_ptr(), self.coef.data_ptr(),
                      self.per, B, self.pred_type, out.data_ptr())
            if j == k - 1:
                break
            x_cur, t_cur = out, torch.clamp(t_next, min=0)
            x2 = torch.cat([x_cur] * nb, 0)
            t2 = torch.cat([t_cur] * nb, 0)
            eps_cu = u.forward(x2, t2, self.in_ctx3[B * 77:(1 + nb) * B * 77], lora=False,
                               added_cond=added(B, (1 + nb) * B))
            eps_c = eps_cu[:B]
            eps_u = eps_cu[B:] if self.apply_cfg else eps_c

    def teacher_step_kernel(self, eps_c, eps_u):
        """x_prev <- DDIM step of the CFG-mixed teacher prediction (T15:1224-1258), one launch."""
        ops._call("pcm_teacher_step", eps_c.data_ptr(), eps_u.data_ptr(), self.noisy.data_ptr(),
                  self.coef.data_ptr(), self.per, self.B, self.pred_type, self.x_prev.data_ptr())

    def loss_kernel(self, eps_s, eps_t):
        """loss, d loss / d eps_student (+ model_pred / target dumps) (T15:1200-1212, 1269-1293)."""
        ops._call("pcm_loss", eps_s.data_ptr(), eps_t.data_ptr(), self.noisy.data_ptr(), self.x_prev.data_ptr(),
                  self.coef.data_ptr(), self.per, self.B, self.loss_type, self.huber_c, self.pred_type,
                  self.loss.data_ptr(), self.d_eps.data_ptr(), ops._p(self.model_pred), ops._p(self.target))

    def optimizer_step(self):
        if self.world > 1 and not self._overlap:
            # ONE collective per step: SUM of the flat LoRA gradient; 1/world is folded into AdamW
            dp.allreduce_flat_grad(self.unet.lora_grad, self.pg)
        self._optimizer_kernels()

    def _optimizer_kernels(self):
        u = self.unet
        g = u.lora_grad
        ops._call("pcm_grad_sumsq", g.data_ptr(), g.numel(), self.sumsq.data_ptr())
        ops._call("pcm_adamw_clip", u.lora_master.data_ptr(), g.data_ptr(), self.exp_avg.data_ptr(),
                  self.exp_avg_sq.data_ptr(), g.numel(), self.opt_state.data_ptr(), self.betas[0],
                  self.betas[1], self.adam_eps, self.wd, self.max_norm, 1.0 / self.world,
                  self.sumsq.data_ptr(), 1)
        if self.ema_master is not None:   # update_ema(target, source, rate): targ = rate*targ + (1-rate)*src
            ops._call("pcm_ema_update", self.ema_master.data_ptr(), u.lora_master.data_ptr(),
                      self.ema_master.numel(), float(self.ema_decay))
        u.refresh_lora()

    def run_eager(self, optimizer=True):
        self.forward_backward()
        if optimizer:
            self.optimizer_step()
        return self.loss

    def capture(self, warmup=2):
        """Capture the iteration into CUDA graph(s) after eager warm-up runs.  Single GPU: one graph
        for forward + backward + optimiser.  Data parallel: graph(forward+backward) -> eager NCCL
        all-reduce -> graph(optimiser) (PCM_NCCL_IN_GRAPH=1 captures the collective too)."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        snap = (self.unet.lora_master.clone(), self.exp_avg.clone(), self.exp_avg_sq.clone(),
                self.opt_state.clone())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self.run_eager()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.graph, self.graph_opt = None, None
        n0 = ops.LAUNCHES["count"]
        in_graph = self.world == 1 or os.environ.get("PCM_NCCL_IN_GRAPH", "0") == "1"
        if in_graph:
            # ONE graph for the whole iteration.  Data parallel default: graph(forward + backward) ->
            # eager NCCL all-reduce -> graph(optimiser).  PCM_NCCL_IN_GRAPH=1 (experimental) captures the
            # bucketed, backward-overlapped all-reduces inside the single graph: it steps correctly on 2
            # GPUs but process-group teardown hung while the graph was
            # alive, so it is not the default; drop `self.graph` before destroy_process_group().
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.run_eager()
            self.graph = g
        else:
            # data parallel: keep the collective outside the graphs (robust across NCCL versions):
            # graph(forward + backward) -> eager all_reduce -> graph(clip + AdamW + LoRA refresh)
            g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            ov, self._overlap = self._overlap, False
            with torch.cuda.graph(g1):
                self.forward_backward()
            with torch.cuda.graph(g2):
                self._optimizer_kernels()
            self._overlap = ov
            self.graph, self.graph_opt = g1, g2
        ops.LAUNCHES["per_step"] = ops.LAUNCHES["count"] - n0
        # the warm-up / capture runs must not count as training steps
        self.unet.lora_master.copy_(snap[0])
        self.exp_avg.copy_(snap[1])
        self.exp_avg_sq.copy_(snap[2])
        self.opt_state.copy_(snap[3])
        if self.ema_master is not None:
            self.ema_master.copy_(snap[0])
        self.unet.lora_grad.zero_()
        self.unet.refresh_lora()
        return self.graph

    def load_inputs(self, latents, noise, index, w, prompt, uncond, text_embeds=None, time_ids=None,
                    non_blocking=True):
        """Copy one batch into the static slots (host pinned or device tensors, NHWC latents).
        text_embeds [B, text_embed_dim] / time_ids [B, 6]: SDXL added conditions."""
        if self.addc:
            if text_embeds is None or time_ids is None:
                raise ValueError("this UNet needs text_embeds and time_ids (added_cond_kwargs)")
            B = self.B
            self.in_text3[:B].copy_(text_embeds, non_blocking=non_blocking)
            self.in_text3[B:2 * B].copy_(text_embeds, non_blocking=non_blocking)
            for i in range(3):
                self.in_time_ids3[i * B:(i + 1) * B].copy_(time_ids, non_blocking=non_blocking)
        self.in_latents.copy_(latents, non_blocking=non_blocking)
        self.in_noise.copy_(noise, non_blocking=non_blocking)
        self.in_index.copy_(index, non_blocking=non_blocking)
        self.in_w.copy_(w, non_blocking=non_blocking)
        self.in_prompt.copy_(prompt.reshape(self.in_prompt.shape), non_blocking=non_blocking)
        self.in_uncond.copy_(uncond.reshape(self.in_uncond.shape), non_blocking=non_blocking)

    def step(self):
        if self.graph is None:
            self.run_eager()
        elif getattr(self, "graph_opt", None) is None:
            self.graph.replay()
        else:
            self.graph.replay()
            dp.allreduce_flat_grad(self.unet.lora_grad, self.pg)
            self.graph_opt.replay()
        return self.loss

    # -- training state (accelerator.save_state / load_state, T15:1080-1105, 1308-1343) -----------
    def state_dict(self):
        """LoRA masters, AdamW moments, (lr, optimiser step) and the optional EMA copy."""
        sd = dict(lora_master=self.unet.lora_master.detach().cpu().clone(),
                  exp_avg=self.exp_avg.cpu().clone(), exp_avg_sq=self.exp_avg_sq.cpu().clone(),
                  opt_state=self.opt_state.cpu().clone())
        if self.ema_master is not None:
            sd["ema_master"] = self.ema_master.cpu().clone()
        return sd

    def load_state_dict(self, sd):
        n = self.unet.lora_master.numel()
        for k in ("lora_master", "exp_avg", "exp_avg_sq"):
            if sd[k].numel() != n:
                raise ValueError(f"checkpoint tensor {k} has {sd[k].numel()} elements, expected {n}")
        self.unet.lora_master.copy_(sd["lora_master"])
        self.exp_avg.copy_(sd["exp_avg"])
        self.exp_avg_sq.copy_(sd["exp_avg_sq"])
        self.opt_state.copy_(sd["opt_state"])
        if self.ema_master is not None:
            self.ema_master.copy_(sd.get("ema_master", sd["lora_master"]))
        self.unet.lora_grad.zero_()
        self.unet.refresh_lora()
