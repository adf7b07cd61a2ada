"""Per-tensor check of the UNet's LoRA gradients against float64 autograd.

For one configuration three gradient sets of sum(eps_student * G) are computed, G a fixed seeded cotangent:
  * ref:  float64 autograd on the operands the product really uses: frozen conv / linear weights, latents,
          context and pooled text embeddings rounded to bf16 (exact properties of the inputs), the fp32 LoRA
          masters, no rounding inside the network;
  * base: the bf16-emulating oracle in float32 with round_grads=True (oracle/unet_ref.py): the error an honest
          bf16 implementation of the same network has;
  * prod: the product's lora_grad_dict() after its merged student + teacher forward (lora_batch = B of 3B
          rows) and backward - the CUDA kernels, or on the CPU their interpretation (tests/ops_interp.py).

Every LoRA tensor k must satisfy both
    rel_L2(prod_k, ref_k) <= RATIO * rel_L2(base_k, ref_k) + REL_FLOOR
    max|prod_k - ref_k|   <= C_MAX * max|base_k - ref_k| + MAX_FLOOR * max|ref_k|
and a tensor whose reference is exactly zero must be exactly zero.  The student rows of the merged forward's
eps are held to the same rule against the LoRA network, the teacher rows against the frozen one.

The bounds are relative to the baseline's error, so they tighten with it: a tensor the bf16 arithmetic
computes to 0.3 % must come out within 0.6 %, whatever the error of the worst tensor.

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit), over every tensor of the SD1.5 / SDXL
configurations of tests/test_lora_grads_gpu.py and the whole-step check: see the constants below.

A 5 % error is only distinguishable from bf16 noise in a tensor whose baseline error is under about 2.5 %:
the rule admits twice the baseline.  The baseline rel-L2 reaches 4.4 % on a few tensors at full width
(up to 9 % in the whole step), so the scaling mutation below is applied to the tensor with the largest
baseline error under SCALE_RESOLVED, and reports how many tensors lie above it.
"""
import contextlib
import statistics
import time
from dataclasses import dataclass, field

import torch

from oracle import unet_ref

BF16 = torch.bfloat16

# rel-L2 rule: the product may have up to twice the error of the bf16 baseline.
RATIO = 2.0
# max-abs rule.  Over the 4 912 tensors of the GPU tests (two runs) the prod / base max ratio has a
# median of 0.96 - 1.04 per configuration and a worst of 2.88 - 2.95 (SDXL, an attn1.to_q B-gradient of
# up_blocks.0); every other configuration stays under 2.6.  4 leaves a 1.36x margin over the worst.
# The rel-L2 ratio has a median of 0.96 - 1.02 and reaches 1.89 at worst (SD1.5 rank 8,
# up_blocks.3...attn1.to_out.0 A-gradient, 1.1e-2 against a baseline of 5.9e-3): a 1.06x margin.
C_MAX = 4.0
# floors, relative to the reference tensor: far below any baseline error (the smallest baseline rel-L2 is
# ~1e-3), they only keep tensors the baseline computes exactly from needing an exact product result.
REL_FLOOR = 1e-4
MAX_FLOOR = 1e-4
SCALE_RESOLVED = 0.025


def bf16_exact(t):
    return t.to(BF16).to(t.dtype)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


@contextlib.contextmanager
def full_fp32():
    """fp32 GEMMs and convolutions really in fp32: cuDNN would otherwise run the baseline's convolutions
    in TF32, whose 10-bit mantissa is coarser than the bf16 arithmetic the baseline stands for."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def ref_params(P, dtype, device):
    """The parameters the product computes with, in `dtype` on `device`: frozen conv / linear weights
    rounded to bf16 (the product's GEMM operands), everything else (fp32 LoRA masters, biases, norm
    affines) as given."""
    out = {}
    for k, v in P.items():
        if ".lora_" not in k and k.endswith(".weight") and v.dim() >= 2:
            v = v.to(BF16)
        out[k] = v.to(device=device, dtype=dtype)
    return out


def make_inputs(ocfg, B, hw, seed):
    """Student rows (B) and teacher rows (2B) with inputs of their own, all bf16-exact, and a bf16-exact
    cotangent G for the student's eps."""
    g = torch.Generator().manual_seed(seed)
    n = 3 * B
    x = bf16_exact(torch.randn(n, 4, hw, hw, generator=g))
    ts = torch.randint(0, 1000, (n,), generator=g)
    ctx = bf16_exact(torch.randn(n, 77, ocfg.cross_attention_dim, generator=g))
    added = None
    if ocfg.addition_embed:
        res = float(hw * 8)
        added = dict(text_embeds=bf16_exact(torch.randn(n, ocfg.text_embed_dim, generator=g)),
                     time_ids=torch.tensor([[res, res, 0.0, 0.0, res, res]] * B +
                                           [[res * 2, res, 8.0, 0.0, res, res * 2]] * (2 * B)).long())
    G = bf16_exact(torch.randn(B, 4, hw, hw, generator=g) / (B * 4 * hw * hw))
    return dict(x=x, ts=ts, ctx=ctx, added=added, G=G, B=B)


def _rows(inp, sl):
    add = None if inp["added"] is None else {k: v[sl] for k, v in inp["added"].items()}
    return inp["x"][sl], inp["ts"][sl], inp["ctx"][sl], add


def oracle_run(ocfg, P, inp, *, dtype, emulate, device):
    """(student eps, teacher eps, LoRA gradients of sum(eps_student * G)) of the oracle network."""
    B = inp["B"]
    Pd = ref_params(P, dtype, device) if not emulate else {k: v.to(device=device, dtype=dtype) for k, v in P.items()}
    lk = unet_ref.lora_keys(Pd)
    for k in lk:
        Pd[k].requires_grad_(True)

    def dev(x, ts, ctx, add):
        add = None if add is None else {k: (v.to(device, dtype) if k == "text_embeds" else v.to(device))
                                        for k, v in add.items()}
        return x.to(device, dtype), ts.to(device), ctx.to(device, dtype), add

    with full_fp32():
        x, ts, ctx, add = dev(*_rows(inp, slice(0, B)))
        eps = unet_ref.UNetRef(ocfg, Pd, use_lora=True, emulate_bf16=emulate, round_grads=emulate)(x, ts, ctx, add)
        (eps * inp["G"].to(device, dtype)).sum().backward()
        grads = {k: Pd[k].grad for k in lk}
        eps = eps.detach()
        del x, ctx, add
        with torch.no_grad():
            x, ts, ctx, add = dev(*_rows(inp, slice(B, 3 * B)))
            eps_t = unet_ref.UNetRef(ocfg, Pd, use_lora=False, emulate_bf16=emulate)(x, ts, ctx, add)
    return eps, eps_t, grads


def product_run(net, inp, device):
    """The merged pass: forward(3B rows, lora_batch=B, save=True), backward(G) of the student rows.
    Returns (student eps, teacher eps, gradient dict, flat lora_grad) in NCHW / oracle layouts."""
    B = inp["B"]
    x, ts, ctx, add = inp["x"], inp["ts"], inp["ctx"], inp["added"]
    added = None if add is None else (add["text_embeds"].to(device, BF16), add["time_ids"].to(device))
    eps = net.forward(_nhwc(x).to(device), ts.to(device), ctx.to(device, BF16).reshape(3 * B * 77, -1), lora=True,
                      save=True, lora_batch=B, added_cond=added)
    net.lora_grad.zero_()
    net.backward(_nhwc(inp["G"]).to(device))
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize()
    eps = _nchw(eps)
    return eps[:B], eps[B:], net.lora_grad_dict(), net.lora_grad


def outside_views(net):
    """Elements of the flat lora_grad no LoRA gradient view covers, and whether the views overlap."""
    cover = torch.zeros(net.lora_grad.numel(), dtype=torch.int32, device=net.lora_grad.device)
    for L in net.lora_layers:
        lo = L.lora
        cover[lo.a_off:lo.a_off + lo.gA.numel()] += 1
        cover[lo.b_off:lo.b_off + lo.gB.numel()] += 1
    return cover == 0, bool((cover > 1).any())


def reset_peak(device):
    torch.cuda.synchronize(device)      # initialises CUDA: the peak of a device not yet in use cannot be reset
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(device)


@dataclass
class GradSets:
    name: str
    prod: dict
    base: dict
    ref: dict
    eps: dict = field(default_factory=dict)     # "student" / "teacher": (prod, base, ref)
    outside_max: float = 0.0                    # max |lora_grad| outside the views
    overlap: bool = False
    peak_gib: float = float("nan")
    wall_s: float = 0.0


def compute(name, ocfg, P, make_net, inp, device):
    """The three gradient sets of one configuration, one network at a time (each freed before the next)."""
    cuda = torch.device(device).type == "cuda"
    if cuda:
        reset_peak(device)
    t0 = time.perf_counter()
    net = make_net()
    e_s, e_t, prod, flat = product_run(net, inp, device)
    outside, overlap = outside_views(net)
    outside_max = flat[outside].abs().max().item() if bool(outside.any()) else 0.0
    e_s, e_t, flat = e_s.clone(), e_t.clone(), None
    del net
    if cuda:
        torch.cuda.empty_cache()
    r_s, r_t, ref = oracle_run(ocfg, P, inp, dtype=torch.float64, emulate=False, device=device)
    if cuda:
        torch.cuda.empty_cache()
    b_s, b_t, base = oracle_run(ocfg, P, inp, dtype=torch.float32, emulate=True, device=device)
    if cuda:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(device) / 2 ** 30 if cuda else float("nan")
    return GradSets(name, prod, base, ref, dict(student=(e_s, b_s, r_s), teacher=(e_t, b_t, r_t)),
                    outside_max, overlap, peak, wall)


@dataclass
class Row:
    key: str
    rel_prod: float
    rel_base: float
    max_prod: float
    max_base: float
    max_ref: float
    ok: bool
    why: str = ""

    @property
    def ratio(self):
        return self.rel_prod / max(self.rel_base, 1e-30)

    @property
    def max_ratio(self):
        return self.max_prod / max(self.max_base, 1e-30)


def check_tensor(key, prod, base, ref):
    r = ref.double()
    dp, db = prod.double().reshape(r.shape) - r, base.double().reshape(r.shape) - r
    mr = r.abs().max().item()
    if mr == 0.0:
        mp = prod.double().abs().max().item()
        return Row(key, 0.0, 0.0, mp, db.abs().max().item(), 0.0, mp == 0.0, "" if mp == 0.0 else "not zero")
    rn = r.norm().item()
    ep, eb = dp.norm().item() / rn, db.norm().item() / rn
    mp, mb = dp.abs().max().item(), db.abs().max().item()
    why = []
    if not ep <= RATIO * eb + REL_FLOOR:
        why.append(f"rel-L2 {ep:.3e} > {RATIO} x {eb:.3e}")
    if not mp <= C_MAX * mb + MAX_FLOOR * mr:
        why.append(f"max {mp:.3e} > {C_MAX} x {mb:.3e}")
    return Row(key, ep, eb, mp, mb, mr, not why, "; ".join(why))


@dataclass
class Report:
    name: str
    rows: list
    eps_rows: list
    sets: GradSets

    @property
    def failures(self):
        bad = [r for r in self.rows + self.eps_rows if not r.ok]
        if self.sets.outside_max != 0.0:
            bad.append(Row("lora_grad outside the views", 0, 0, self.sets.outside_max, 0, 0, False, "not zero"))
        if self.sets.overlap:
            bad.append(Row("lora_grad views", 0, 0, 0, 0, 0, False, "overlap"))
        return bad

    def summary(self):
        live = [r for r in self.rows if r.max_ref > 0]
        ratios = [r.ratio for r in live]
        mratios = [r.max_ratio for r in live]
        worst = max(live, key=lambda r: r.ratio)
        worst_m = max(live, key=lambda r: r.max_ratio)
        s = self.sets
        eps = " ".join(f"eps {k} {r.rel_prod:.2e}/{r.rel_base:.2e}" for k, r in zip(("student", "teacher"), self.eps_rows))
        return (f"[{self.name}] {len(self.rows)} tensors ({len(self.rows) - len(live)} zero) | rel-L2 prod/base median "
                f"{statistics.median(ratios):.3f} worst {worst.ratio:.3f} ({worst.key}: {worst.rel_prod:.2e} vs "
                f"{worst.rel_base:.2e}) | max prod/base median {statistics.median(mratios):.3f} worst "
                f"{worst_m.max_ratio:.3f} ({worst_m.key}) | base rel-L2 max {max(r.rel_base for r in live):.2e} | "
                f"{eps} | peak {s.peak_gib:.1f} GiB | {s.wall_s:.1f} s")


def check(sets, prod=None):
    """Report of the rule over every LoRA tensor (of `prod`, default sets.prod) and both eps row sets."""
    prod = sets.prod if prod is None else prod
    assert set(prod) == set(sets.ref), sorted(set(prod) ^ set(sets.ref))[:4]
    rows = [check_tensor(k, prod[k], sets.base[k], sets.ref[k]) for k in sorted(sets.ref)]
    eps_rows = [check_tensor("eps " + k, *v) for k, v in sets.eps.items()]
    return Report(sets.name, rows, eps_rows, sets)


def assert_passes(report):
    print(report.summary())
    bad = report.failures
    assert not bad, f"{report.name}: {len(bad)} failing: " + "; ".join(f"{r.key}: {r.why}" for r in bad[:8])


# ---------------------------------------------------------------------------------------------------------
# mutations: plausible plan bugs applied to a passing gradient set; the check must reject each
# ---------------------------------------------------------------------------------------------------------
def _worst_base(sets, keys):
    return max(keys, key=lambda k: check_tensor(k, sets.base[k], sets.base[k], sets.ref[k]).rel_base)


def _conv3_a_keys(sets):
    """3x3 conv A-gradients whose tap (0, 0) carries at least 2 % of the tensor's squared norm (at a 1 x 1
    level every tap but the centre reads padding only, and zeroing it would change nothing)."""
    out = []
    for k, v in sets.ref.items():
        if k.endswith("lora_A.weight") and v.dim() == 4 and v.shape[-1] == 3 and v.abs().max() > 0:
            if v[:, :, 0, 0].pow(2).sum() >= 0.02 * v.pow(2).sum():
                out.append(k)
    return out


def mutations(sets):
    """{name: mutated copy of sets.prod}."""
    g = sets.prod
    live = [k for k in g if sets.ref[k].abs().max() > 0]
    out = {}
    q = next(k for k in sorted(g) if k.endswith("attn1.to_q.lora_A.weight"))
    kk = q.replace("to_q", "to_k")
    out["swap attn1.to_q / to_k A-gradients"] = {**g, q: g[kk], kk: g[q]}
    base = {k: check_tensor(k, sets.base[k], sets.base[k], sets.ref[k]).rel_base for k in live}
    resolved = [k for k in live if base[k] < SCALE_RESOLVED]
    k = max(resolved, key=base.get)
    out[f"scale {k} (baseline rel-L2 {base[k]:.2e}; {len(live) - len(resolved)} of {len(live)} tensors have "
        f"more) by 1.05"] = {**g, k: g[k] * 1.05}
    z = max(live, key=base.get)
    c = _worst_base(sets, _conv3_a_keys(sets))
    t = g[c].clone()
    t[:, :, 0, 0] = 0
    out[f"zero tap (0, 0) of {c}"] = {**g, c: t}
    r, cin = g[c].shape[:2]
    out[f"read {c} OHWI as OIHW"] = {**g, c: g[c].permute(0, 2, 3, 1).reshape(r, cin, 3, 3)}
    out[f"zero {z}"] = {**g, z: torch.zeros_like(g[z])}
    return out


def assert_mutations_rejected(sets):
    for name, prod in mutations(sets).items():
        rep = check(sets, prod)
        bad = [r for r in rep.rows if not r.ok]
        print(f"[{sets.name}] mutation '{name}': rejected by {len(bad)} tensor(s)"
              + (f", e.g. {bad[0].key}: {bad[0].why}" if bad else ""))
        assert bad, f"{sets.name}: the check accepts the mutation '{name}'"
