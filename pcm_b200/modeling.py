"""Call-shape mirror of the model objects the reference loop uses (train_pcm_lora_sd15.py):

    unet(noisy_model_input, start_timesteps, timestep_cond=None,
         encoder_hidden_states=prompt_embeds.float(), added_cond_kwargs=...).sample      (:1192-1198)
    teacher_unet(...).sample                                                              (:1219-1223)

`UNet2DConditionModel` wraps the CUDA network (`pcm_b200.unet.UNetB200`, NHWC bf16 inside) behind
diffusers' NCHW signature: CUDA tensors in, `.sample` fp32 NCHW out (accelerate's autocast wrapper
converts outputs to fp32, SURVEY App. A1).  `use_lora=False` gives the frozen teacher on the SAME
weights.  The layout change of the 4-channel latents is a torch permute (plumbing, 64 KB / sample);
every FLOP runs in libpcm_b200.so.  There is no CPU fallback.
"""
from dataclasses import dataclass

import torch

from .unet import UNetB200


@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor


class UNet2DConditionModel:
    def __init__(self, net: UNetB200, use_lora=True):
        self.net, self.use_lora = net, use_lora
        self.config = net.cfg
        self.training = use_lora

    # -- the slice of the nn.Module / peft API the training script touches -----------------------
    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def requires_grad_(self, flag=True):
        return self

    def parameters(self):
        """Trainable parameters: the flat LoRA buffer (only LoRA tensors require grad, T15:885)."""
        return [self.net.lora_master] if self.use_lora and self.net.has_lora else []

    def enable_gradient_checkpointing(self):
        """No recompute is needed: the bs 8 SD1.5 step fits an 80 GB H100 without it; accepted for API parity."""

    def enable_xformers_memory_efficient_attention(self):
        """Attention always runs the library's flash kernels; accepted for API parity."""

    def get_peft_model_state_dict(self):
        return self.net.lora_state_dict()

    def __call__(self, sample, timestep, timestep_cond=None, encoder_hidden_states=None,
                 added_cond_kwargs=None, return_dict=True, save_for_backward=False):
        if timestep_cond is not None:
            raise ValueError("timestep_cond is not used by the SD1.5 UNet (time_cond_proj_dim=None)")
        if encoder_hidden_states is None:
            raise ValueError("encoder_hidden_states is required (CrossAttn blocks)")
        if not sample.is_cuda:
            raise RuntimeError("pcm_b200 needs CUDA tensors (no CPU fallback)")
        B = sample.shape[0]
        ts = torch.as_tensor(timestep, device=sample.device).to(torch.int64).reshape(-1)
        if ts.numel() == 1:
            ts = ts.expand(B)
        x = sample.float().permute(0, 2, 3, 1).contiguous()
        ctx = encoder_hidden_states.to(device=sample.device, dtype=torch.bfloat16).reshape(B * encoder_hidden_states.shape[1], -1)
        eps = self.net.forward(x, ts.contiguous(), ctx.contiguous(), lora=self.use_lora, save=save_for_backward)
        out = eps.permute(0, 3, 1, 2).contiguous()
        return UNet2DConditionOutput(sample=out) if return_dict else (out,)

    def backward(self, d_sample):
        """Gradient of a scalar w.r.t. `.sample` (NCHW) -> LoRA gradients in net.lora_grad."""
        self.net.backward(d_sample.float().permute(0, 2, 3, 1).contiguous())
