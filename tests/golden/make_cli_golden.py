"""Extract the command-line surface of the reference training script (flag names, defaults,
actions, types) by AST - nothing is imported or executed - into tests/golden/cli_flags.json.
Run in the build container (the reference tree is not available on the GPU box):
    python tests/golden/make_cli_golden.py
"""
import ast
import json
import os

# a checkout of G-U-N/Phased-Consistency-Model (read only), given by PCM_REFERENCE
REF = os.path.join(os.environ["PCM_REFERENCE"], "code/text_to_image_sd15/train_pcm_lora_sd15.py")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cli_flags.json")


def lit(node):
    try:
        return ast.literal_eval(node)
    except Exception:
        return {"expr": ast.unparse(node)}


def main():
    tree = ast.parse(open(REF).read())
    flags = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            names = [a.value for a in node.args if isinstance(a, ast.Constant) and isinstance(a.value, str)]
            if not names or not names[0].startswith("--"):
                continue
            kw = {k.arg: k.value for k in node.keywords}
            entry = {"line": node.lineno}
            if "default" in kw:
                entry["default"] = lit(kw["default"])
            if "action" in kw:
                entry["action"] = lit(kw["action"])
            if "type" in kw:
                entry["type"] = ast.unparse(kw["type"])
            if "nargs" in kw:
                entry["nargs"] = lit(kw["nargs"])
            if "choices" in kw:
                entry["choices"] = lit(kw["choices"])
            if "required" in kw:
                entry["required"] = lit(kw["required"])
            flags[names[0]] = entry
    json.dump({"source": "code/text_to_image_sd15/train_pcm_lora_sd15.py", "flags": flags}, open(OUT, "w"),
              indent=1, sort_keys=True)
    print(len(flags), "flags ->", OUT)


if __name__ == "__main__":
    main()
