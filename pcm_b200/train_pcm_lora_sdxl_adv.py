#!/usr/bin/env python
"""`train_pcm_lora_sdxl_adv` entry point on the CUDA path (SURVEY section 8f-2).

Same command line as code/text_to_image_sdxl/train_pcm_lora_sdxl_adv.py (the SD1.5
flags plus --adv_weight, --adv_lr, --train_shards_path_or_url, --use_fix_crop_and_size) driving the
SDXL UNet (3 levels, transformer depth 1 / 2 / 10, 64-wide heads, 2048-d context, Linear projections,
`added_cond_kwargs` text_time embedding, zero unconditional embeddings).  The consistency-distillation
step (student / teacher CFG solve / target / Huber-L2 / AdamW) runs through the same fused kernels as
SD1.5.  NOT implemented: the adversarial term (Discriminator over the teacher backbone,
discriminator_sdxl.py) - the script therefore requires `--adv_weight 0` and says so; everything else
of the step is the reference's (TXL:1277-1603 minus the d_loss / g_loss branches).
"""
from . import config
from . import train_pcm_lora_sd15 as base


def _extra(p):
    p.add_argument("--adv_weight", default=0.1, type=float)
    p.add_argument("--adv_lr", default=1e-5, type=float)
    p.add_argument("--train_shards_path_or_url", type=str, default=None)
    p.add_argument("--use_fix_crop_and_size", action="store_true")


def parse_args(argv=None):
    args = base.parse_args(argv, extra=_extra)
    if args.adv_weight != 0:
        raise ValueError("the adversarial consistency loss (discriminator_sdxl.Discriminator) is not implemented "
                         "on the CUDA path: pass --adv_weight 0 to run the consistency-distillation step alone")
    args._base_cfg = config.SDXL
    return args


def main(args):
    return base.main(args)


if __name__ == "__main__":
    main(parse_args())
