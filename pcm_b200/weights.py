"""Weight sources for the UNet: seeded synthetic initialisation (no pretrained checkpoint is
available offline) and state-dict helpers using diffusers / peft key names, so a real
`runwayml/stable-diffusion-v1-5` UNet state dict can be dropped in unchanged
(train_pcm_lora_sd15.py:840-852, 866-885)."""
import torch

from .config import UNetConfig, is_lora_target, layer_table


def synthetic_state_dict(cfg: UNetConfig, seed: int = 0, lora_b_std: float = 0.02):
    """nn.Conv2d / nn.Linear default init U(-1/sqrt(fan_in), 1/sqrt(fan_in)); norm affine (1, 0);
    LoRA A kaiming-uniform(a=sqrt(5)) like peft, LoRA B ~ N(0, lora_b_std) (peft uses zeros; a
    non-zero B keeps every LoRA GEMM and gradient numerically live for benchmarking)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def uni(shape, bound):
        return (torch.rand(shape, generator=g) * 2 - 1) * bound

    r = cfg.lora_rank
    for name, kind, cin, cout, k in layer_table(cfg):
        if kind in ("gn", "ln"):
            sd[name + ".weight"] = torch.ones(cout)
            sd[name + ".bias"] = torch.zeros(cout)
            continue
        if kind == "conv":
            fan = cin * k * k
            sd[name + ".weight"] = uni((cout, cin, k, k), fan ** -0.5)
            sd[name + ".bias"] = uni((cout,), fan ** -0.5)
        else:
            sd[name + ".weight"] = uni((cout, cin), cin ** -0.5)
            if kind == "linear":
                sd[name + ".bias"] = uni((cout,), cin ** -0.5)
        if is_lora_target(name):
            if kind == "conv":
                sd[name + ".lora_A.weight"] = uni((r, cin, k, k), (cin * k * k) ** -0.5)
                sd[name + ".lora_B.weight"] = torch.randn((cout, r, 1, 1), generator=g) * lora_b_std
            else:
                sd[name + ".lora_A.weight"] = uni((r, cin), cin ** -0.5)
                sd[name + ".lora_B.weight"] = torch.randn((cout, r), generator=g) * lora_b_std
    return sd


def to_peft_keys(lora_sd):
    """`<module>.lora_A.weight` -> peft adapter key `base_model.model.<module>.lora_A.weight`
    (what get_peft_model_state_dict returns, train_pcm_lora_sd15.py:921-927)."""
    return {"base_model.model." + k: v for k, v in lora_sd.items()}


def to_kohya_keys(lora_sd, lora_alpha, dtype=torch.float32):
    """Kohya-style dict as built by get_module_kohya_state_dict (train_pcm_lora_sd15.py:52-72)."""
    out = {}
    for k, w in lora_sd.items():
        module = k.rsplit(".lora_", 1)[0]
        which = "lora_down" if ".lora_A." in k else "lora_up"
        base = "lora_unet_" + module.replace(".", "_")
        out[f"{base}.{which}.weight"] = w.to(dtype)
        if which == "lora_down":
            out[f"{base}.alpha"] = torch.tensor(lora_alpha).to(dtype)
    return out
