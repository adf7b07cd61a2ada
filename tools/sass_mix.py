"""Instruction mix of the library's kernels, read from `cuobjdump -sass` (no GPU needed).

For every kernel whose mangled name matches the pattern it prints the opcode counts of the whole kernel
and of each loop (a backward branch and the instructions from its target to it) that holds at least
--min-loop instructions.  A loop's count is static: instructions behind a branch inside the loop (the
forward's skipped O rescale, for one) count as if they ran every iteration.  The columns relate the
exp-related opcodes to the MUFU.EX2 count, so a denormal-handling compare / multiply around each exp,
or a select per score element, shows up as a ratio near 1 or 2.

Usage: python tools/sass_mix.py [--lib pcm_b200/lib/libpcm_b200.so | --sass FILE] [--kernel REGEX]
                                [--min-loop N] [--all-ops]"""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNC = re.compile(r"^\s*Function : (\S+)")
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?);")
BRANCH = re.compile(r"^(?:@!?U?P\w+\s+)?BRA(?:\.\S+)?\s+(?:.*?)(0x[0-9a-f]+)")
# opcodes the softmax diet is about, shown as columns; the rest are summed as "other"
COLUMNS = ["MUFU.EX2", "FSETP", "FSEL", "FMUL", "FADD", "FFMA", "FMNMX", "F2FP", "SHFL", "HGMMA", "VOTE"]


def opcode(text):
    """Opcode of one SASS instruction: the mnemonic without modifiers, except MUFU keeps its function."""
    t = re.sub(r"^@!?U?P\w+\s+", "", text.strip())
    op = t.split()[0] if t else ""
    return op if op.startswith("MUFU.") else op.split(".")[0]


def parse(sass):
    """{kernel: [(address, instruction text)]} in program order."""
    kernels, cur = {}, None
    for line in sass.splitlines():
        m = FUNC.match(line)
        if m:
            cur = kernels.setdefault(m.group(1), [])
            continue
        m = INSN.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2)))
    return kernels


def loops(insns):
    """(first index, last index) of every loop, outermost first: a branch back to an earlier address.
    ptxas places the retry of a failed mbarrier wait after the kernel's exits and branches back from
    there; such a range holds an EXIT and is not a loop of the program, so it is left out."""
    index = {a: i for i, (a, _) in enumerate(insns)}
    out = []
    for i, (a, text) in enumerate(insns):
        m = BRANCH.match(text.strip())
        if not m:
            continue
        t = int(m.group(1), 16)
        if t <= a and t in index and not any(opcode(x) == "EXIT" for _, x in insns[index[t]:i]):
            out.append((index[t], i))
    return sorted(set(out), key=lambda r: (r[0], -r[1]))


def mix(insns):
    return collections.Counter(opcode(t) for _, t in insns if opcode(t) != "NOP")


def row(name, c, all_ops):
    total = sum(c.values())
    cells = [f"{c.get(k, 0):6d}" for k in COLUMNS]
    other = total - sum(c.get(k, 0) for k in COLUMNS)
    ex2 = c.get("MUFU.EX2", 0)
    ratio = f"  FSETP/EX2 {c.get('FSETP', 0) / ex2:4.2f}  FSEL/EX2 {c.get('FSEL', 0) / ex2:4.2f}" if ex2 else ""
    line = f"  {name:<22s}{total:7d}" + "".join(cells) + f"{other:7d}" + ratio
    if all_ops:
        line += "\n      " + ", ".join(f"{k} {v}" for k, v in sorted(c.items(), key=lambda kv: -kv[1]))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", default=os.path.join(ROOT, "pcm_b200", "lib", "libpcm_b200.so"))
    ap.add_argument("--sass", default=None, help="read this cuobjdump -sass listing instead of the library")
    ap.add_argument("--kernel", default=r"attn_(fwd|bwd)_wg_kernel", help="regex on the mangled kernel name")
    ap.add_argument("--min-loop", type=int, default=200, help="smallest loop (instructions) to report")
    ap.add_argument("--all-ops", action="store_true", help="also list every opcode of each row")
    args = ap.parse_args()
    if args.sass:
        with open(args.sass) as f:
            sass = f.read()
    else:
        tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                         "cuobjdump")
        sass = subprocess.run([tool, "-sass", args.lib], check=True, capture_output=True, text=True).stdout
    pat = re.compile(args.kernel)
    header = f"  {'':<22s}{'total':>7s}" + "".join(f"{k.split('.')[-1]:>6s}" for k in COLUMNS) + f"{'other':>7s}"
    found = False
    for name, insns in parse(sass).items():
        if not pat.search(name):
            continue
        found = True
        print(name)
        print(header)
        print(row("kernel", mix(insns), args.all_ops))
        for lo, hi in loops(insns):
            body = insns[lo:hi + 1]
            if len(body) >= args.min_loop:
                print(row(f"loop {insns[lo][0]:#06x}-{insns[hi][0]:#06x}", mix(body), args.all_ops))
        print()
    if not found:
        sys.exit(f"no kernel matches {args.kernel!r}")


if __name__ == "__main__":
    main()
