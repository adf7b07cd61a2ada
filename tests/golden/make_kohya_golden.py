"""Golden key mapping of the reference's kohya export: `get_module_kohya_state_dict`
(train_pcm_lora_sd15.py:52-72) is AST-extracted and executed verbatim; only its peft call is
stubbed (peft is not installed) with the adapter-key layout peft 0.9.0 returns,
`base_model.model.<module>.lora_{A,B}.weight`.  Writes tests/golden/kohya_keys.json.
    python tests/golden/make_kohya_golden.py
"""
import ast
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
# a checkout of G-U-N/Phased-Consistency-Model (read only), given by PCM_REFERENCE
REF = os.path.join(os.environ["PCM_REFERENCE"], "code/text_to_image_sd15/train_pcm_lora_sd15.py")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kohya_keys.json")


def main():
    from pcm_b200 import config
    tree = ast.parse(open(REF).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "get_module_kohya_state_dict")
    modules = [n for n, kind, *_ in config.layer_table(config.SD15) if config.is_lora_target(n)]
    peft_sd = {}
    for m in modules:
        peft_sd[f"base_model.model.{m}.lora_A.weight"] = torch.zeros(1)
        peft_sd[f"base_model.model.{m}.lora_B.weight"] = torch.zeros(1)
    env = {"torch": torch, "get_peft_model_state_dict": lambda module, adapter_name="default": peft_sd}
    exec(compile(ast.Module([fn], []), REF, "exec"), env)
    module = types.SimpleNamespace(peft_config={"default": types.SimpleNamespace(lora_alpha=8)})
    out = env["get_module_kohya_state_dict"](module, "lora_unet", torch.float32)
    json.dump({"modules": modules, "kohya_keys": sorted(out.keys()),
               "alpha": float(next(v for k, v in out.items() if k.endswith(".alpha")))}, open(OUT, "w"), indent=0)
    print(len(modules), "LoRA modules ->", len(out), "kohya keys")


if __name__ == "__main__":
    main()
