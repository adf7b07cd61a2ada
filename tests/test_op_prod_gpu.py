"""Every distinct GroupNorm, LayerNorm, glue and optimiser launch of the real training steps, on the GPU
against float64, and the edges their kernels and host checks are written for.

tests/golden/op_specs.json.gz holds one pointer-free spec per launch class of the SD1.5 (batch 8, 64x64
latents: the benchmark), SDXL, gradient-checkpointing, rank 8 / 32 and EMA + two-substep steps;
test_op_specs_cpu.py keeps it equal to the plan.  Each class is materialised into NaN-poisoned buffers
(TAIL guard bytes after each), launched through the C ABI with exactly the recorded scalars, compared with
op_spec.reference under its derived bound (bit for bit where the op is exact), and every byte outside the
output windows must be unchanged.  GroupNorm, the gradient norm and AdamW must reproduce their results bit
for bit on a second launch and leave their counters at zero.  A class met in several configurations runs
once."""
import math
import os
import time

import pytest
import torch

import op_spec as O

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
_SPECS = O.trace.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "op_specs.json.gz"))
CLASSES, COUNTS = {}, {}
for _name, _specs in _SPECS.items():
    COUNTS[_name] = len(_specs)
    for _i, _s in enumerate(_specs):
        CLASSES.setdefault(O.launch_class(_s), (f"{_name}-{_i}-{_s['op'][4:]}", _s))
CASES = list(CLASSES.values())
WORST = {}
PEAK = {}                  # op -> largest device memory peak of one production launch test (bytes)
T0 = time.time()


def _lib():
    from pcm_b200 import _lib
    return _lib.lib()


def restore(T, before):
    for b, b0 in zip(T.bufs, before.bufs):
        b.copy_(b0)


def outputs(spec, T):
    """Copies of the bytes of every output window (for bitwise reproducibility)."""
    return [T.bufs[lab][off // 2:(off + n + 1) // 2].clone() for lab, off, n in O.out_windows(spec)]


def run(spec, T, before=None):
    """Launch, check against the reference and the guards; returns the worst err / bound per family."""
    before = before or T.snapshot()
    rc = O.launch(spec, T)
    assert rc == 0, _lib().pcm_last_error().decode()
    torch.cuda.synchronize()
    worst = O.check(spec, before, T)
    O.guards(spec, T, before)
    if spec["op"] in O.GN_OPS:
        assert not T.ws[:4 * 3 * O.GN_MAX_B].any(), "the GroupNorm kernels must leave all three counter arrays at zero"
    for k, v in worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    return worst


def run_twice(spec, T):
    """run, then the same launch from the same inputs again: bit-identical outputs."""
    before = T.snapshot()
    run(spec, T, before)
    o1 = outputs(spec, T)
    restore(T, before)
    run(spec, T, before)
    for a, b in zip(o1, outputs(spec, T)):
        assert torch.equal(a, b), f"{spec['op']}: a second launch on the same inputs differs"


def test_workspace_size_matches_the_library(cuda):
    lib = _lib()
    for B, HW, C in ((24, 4096, 320), (2, 16384, 320), (6, 16384, 640), (8, 64, 2560), (1, 1000, 96), (1024, 64, 320)):
        assert lib.pcm_groupnorm_ws_bytes(B, HW, C, 32) == O.gn_ws_bytes(B, HW, C, 32), (B, HW, C)
    assert lib.pcm_groupnorm_ws_bytes(1, 64, 2568, 32) == -1
    assert lib.pcm_num_sms() == O.NUM_SMS, "the recorded plans were tiled for 132 SMs"


@pytest.mark.parametrize("spec", [c[1] for c in CASES], ids=[c[0] for c in CASES])
def test_production_launch(cuda, spec):
    torch.cuda.reset_peak_memory_stats()
    _production(cuda, spec)
    PEAK[spec["op"]] = max(PEAK.get(spec["op"], 0), torch.cuda.max_memory_allocated())


def _production(cuda, spec):
    T = O.materialise(spec, cuda, seed=len(spec["spans"]))
    if spec["op"] in O.GN_OPS or spec["op"] in ("pcm_grad_sumsq", "pcm_lora_refresh"):
        run_twice(spec, T)
    elif spec["op"] == "pcm_adamw_clip":
        run_twice(spec, T)
        run(spec, T)                 # the second update, from the device-side state: step 2
        assert float(T.view("state", F32, 2)[1]) == 2.0
    else:
        run(spec, T)


def _fwd_over(spec, B):
    a = dict(spec["args"])
    a.pop("part_B")
    a["B"] = B
    return O.make_spec("pcm_groupnorm_fwd", **{k: (True if isinstance(v, list) else v) for k, v in a.items()})


PARTS = sorted({(s["args"]["B"], s["args"]["part_B"], s["args"]["HW"], s["args"]["C1"], s["args"]["C2"])
                for specs in _SPECS.values() for s in specs if s["op"] == "pcm_groupnorm_fwd_part"})


@pytest.mark.parametrize("B,part_B,HW,C1,C2", PARTS)
def test_fwd_part_equals_the_leading_rows_of_the_full_launch(cuda, B, part_B, HW, C1, C2):
    spec = next(s for specs in _SPECS.values() for s in specs if s["op"] == "pcm_groupnorm_fwd_part"
                and (s["args"]["B"], s["args"]["part_B"], s["args"]["HW"], s["args"]["C1"], s["args"]["C2"]) == (B, part_B, HW, C1, C2))
    full = _fwd_over(spec, part_B)
    Tf = O.materialise(full, cuda, seed=1)
    run(full, Tf)
    Tp = O.materialise(spec, cuda, seed=2)
    for k in ("x1", "x2", "gamma", "beta"):
        if spec["args"][k]:
            n = Tp.view(k, torch.uint8).numel()
            Tp.view(k, torch.uint8).copy_(Tf.view(k, torch.uint8)[:n])
    run(spec, Tp)
    C = C1 + C2
    assert torch.equal(Tp.view("out", torch.int16, B * HW * C), Tf.view("out", torch.int16, B * HW * C))
    assert torch.equal(Tp.view("stats", torch.int32, B * 64), Tf.view("stats", torch.int32, B * 64))


# ---------------------------------------------------------------------------------------------
# edges beyond production
# ---------------------------------------------------------------------------------------------
def gn(op="pcm_groupnorm_fwd", C1=320, C2=0, B=2, HW=64, G=32, eps=1e-5, silu=1, add=True, colsum=True):
    if op == "pcm_groupnorm_bwd":
        return O.make_spec(op, dy=True, x1=True, x2=True if C2 else None, C1=C1, C2=C2, B=B, HW=HW, G=G, gamma=True, beta=True,
                           eps=eps, silu=silu, stats=True, red=True, add=True if add else None, dx1=True,
                           dx2=True if C2 else None, colsum=True if colsum else None)
    return O.make_spec(op, x1=True, x2=True if C2 else None, C1=C1, C2=C2, B=B, HW=HW, G=G, gamma=True, beta=True, eps=eps,
                       silu=silu, out=True, stats=True)


GN_EDGES = {
    "C2560_split": dict(C1=1280, C2=1280, B=2, HW=64),        # kGnMaxC
    "nblk128_B1": dict(C1=320, B=1, HW=16384),                # 128 blocks of one image: the stage cap
    "short_last_block": dict(C1=320, B=3, HW=1000),
    "B1": dict(C1=640, B=1, HW=4096),
    "cpg3": dict(C1=40, C2=56, B=2, HW=256),                  # one 8-channel vector spans three groups
    "cpg60_straddle": dict(C1=1280, C2=640, B=2, HW=256),     # groups straddle x1 / x2
    "eps1e-6_nosilu": dict(C1=320, B=2, HW=1024, eps=1e-6, silu=0),
}


@pytest.mark.parametrize("name", list(GN_EDGES))
def test_groupnorm_edges(cuda, name):
    run_twice(gn(**GN_EDGES[name]), O.materialise(gn(**GN_EDGES[name]), cuda, 3))
    s = gn("pcm_groupnorm_bwd", **GN_EDGES[name])
    run_twice(s, O.materialise(s, cuda, 4))


@pytest.mark.parametrize("add,colsum", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_groupnorm_backward_add_and_colsum(cuda, add, colsum):
    s = gn("pcm_groupnorm_bwd", C1=640, C2=640, B=3, HW=256, add=add, colsum=colsum)
    run_twice(s, O.materialise(s, cuda, 5))


@pytest.mark.parametrize("k", [100.0, 1000.0])
def test_groupnorm_outlier_pivot(cuda, k):
    """Pixel 0 of every image is a k-sigma outlier, the pivot of the kernel's shifted sums.  The derived
    bound (gn_stats_bound) widens with mean (x - pivot)^2, to a few per cent of rstd at 1000 sigma, so on
    top of it the statistics must stay where a bf16 output cannot see them: mean and rstd errors of at
    most 2^-12 of sigma and of rstd move a normalised value by at most 1/16 of its bf16 rounding (2^-8)."""
    s = gn(C1=320, B=2, HW=4096)
    T = O.materialise(s, cuda, 6)
    x = T.view("x1", BF16, 2 * 4096 * 320).view(2, 4096, 320)
    x[:, 0] = (x[:, 0].float() + k).to(BF16)
    before = T.snapshot()
    run(s, T, before)
    ref = O.gn_stats64(before, s["args"]["eps"])
    st = T.view("stats", F32, 2 * 2 * 32).view(2, 32, 2).double()
    dm = float(((st[..., 0] - ref[..., 0]).abs() * ref[..., 1]).max())
    dr = float(((st[..., 1] - ref[..., 1]).abs() / ref[..., 1]).max())
    print(f"\n  outlier pivot {k:.0f} sigma: mean error {dm:.2e} sigma, rstd error {dr:.2e} relative")
    assert dm <= 2.0 ** -12 and dr <= 2.0 ** -12, (dm, dr)


def ln(fwd, M, C, stats=True, add=True):
    if fwd:
        return O.make_spec("pcm_layernorm_fwd", x=True, M=M, C=C, gamma=True, beta=True, eps=1e-5, out=True, stats=stats or None)
    return O.make_spec("pcm_layernorm_bwd", dy=True, x=True, M=M, C=C, gamma=True, stats=True, add=add or None, dx=True)


def _ln_rows_per_grid(C):
    lpr = 8 if C // 8 <= 40 else (16 if C // 8 <= 80 else 32)
    return 4 * O.NUM_SMS * 8 * (32 // lpr)


@pytest.mark.parametrize("C", [320, 328, 640, 648, 1280])
@pytest.mark.parametrize("M", ["1", "37", "3strides"])
def test_layernorm_edges(cuda, C, M):
    m = {"1": 1, "37": 37, "3strides": 3 * _ln_rows_per_grid(C) + 5}[M]
    for i, s in enumerate((ln(True, m, C), ln(True, m, C, stats=False), ln(False, m, C), ln(False, m, C, add=False))):
        run(s, O.materialise(s, cuda, i))


@pytest.mark.parametrize("C,H,W,bias,sgn", [(8, 5, 7, True, 1), (320, 9, 11, True, 1), (320, 1, 1, False, -1),
                                             (8, 1, 1, True, -1), (320, 16, 16, False, -1)])
def test_conv_c4_edges(cuda, C, H, W, bias, sgn):
    s = O.make_spec("pcm_conv3x3_c4", x=True, B=2, H=H, W=W, C=C, w=True, bias=bias or None, sgn=sgn, round_in=int(sgn > 0), out=True)
    run(s, O.materialise(s, cuda, 7))


def test_geglu_edges(cuda):
    for fwd in (True, False):
        for M, Fh in ((3, 8), (1000, 2560)):
            s = O.make_spec("pcm_geglu_fwd", u=True, M=M, F=Fh, out=True) if fwd else \
                O.make_spec("pcm_geglu_bwd", dgg=True, u=True, M=M, F=Fh, du=True)
            T = O.materialise(s, cuda, 8)
            u = T.view("u", BF16, 2 * M * Fh).view(M, 2, Fh)
            u[:, 1, ::3] = 8.0                        # erf saturates
            u[:, 1, 1::3] = -8.0
            run(s, T)


def test_cast_specials(cuda):
    s = O.make_spec("pcm_cast_f32_bf16", x=True, n=4097, out=True)
    T = O.materialise(s, cuda, 9)
    x = T.view("x", F32, 4097)
    sp = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e-40, -1e-40, 2.0 ** -133, 0.0, -0.0,
                       1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 3.3895e38, -3.3895e38], device=cuda)
    x[:len(sp)] = sp                                  # ties at 1 + 2^-8 round to even in both directions
    x[-3:] = sp[-3:]
    run(s, T)


@pytest.mark.parametrize("n", [1, 3, 4 * 1000 + 1, 4 * 1000 + 2, 4 * 1000 + 3, 4 * 256 * 4 * O.NUM_SMS * 3 + 3])
def test_sumsq_sizes(cuda, n):
    s = O.make_spec("pcm_grad_sumsq", g=True, n=n, out=True)
    run_twice(s, O.materialise(s, cuda, 10))


@pytest.mark.parametrize("case", ["clip", "noclip", "max_norm0", "world2", "keep_grad", "zero_grad_values"])
def test_adamw_edges(cuda, case):
    kw = dict(beta1=0.9, beta2=0.999, eps=1e-8, wd=0.01, max_norm=1.0, inv_world=1.0, zero_grad=1)
    if case == "max_norm0":
        kw["max_norm"] = 0.0
    if case == "world2":
        kw["inv_world"] = 0.5
    if case == "keep_grad":
        kw["zero_grad"] = 0
    s = O.make_spec("pcm_adamw_clip", p=True, g=True, m=True, v=True, n=1000003, state=True, sumsq=True, **kw)
    T = O.materialise(s, cuda, 11)
    g = T.view("g", F32, 1000003)            # N(0, 1e-3^2): a norm of about 1, as large as max_norm
    g.mul_(1e-3 if case == "noclip" else 10.0)
    if case == "zero_grad_values":
        g.zero_()
        T.view("m", F32, 1000003).zero_()
        T.view("v", F32, 1000003).zero_()
    # the sum of squares of the gradient summed over 1 / inv_world ranks, each holding g
    T.view("sumsq", F64, 1)[0] = O.sumsq64(g) / kw["inv_world"] ** 2
    norm = math.sqrt(float(T.view("sumsq", F64, 1)[0])) * kw["inv_world"]
    if case in ("clip", "world2"):
        assert norm > 2 * kw["max_norm"]
    if case == "noclip":
        assert norm < kw["max_norm"] / 2
    run_twice(s, T)
    run(s, T)


# ---------------------------------------------------------------------------------------------
# rejections: a non-zero return with a message, nothing launched
# ---------------------------------------------------------------------------------------------
def _rejected(spec, T, message, **over):
    """The launch returns non-zero with `message`, and no buffer changes.  A rejection of another kind is
    provoked first, so a stale message cannot pass for this one."""
    lib = _lib()
    assert lib.pcm_geglu_fwd(None, 1, 3, None, None) != 0
    assert "geglu" in lib.pcm_last_error().decode()
    before = T.snapshot()
    rc = O.launch(spec, T, **over)
    torch.cuda.synchronize()
    assert rc != 0
    msg = lib.pcm_last_error().decode()
    assert message in msg, f"rejected with {msg!r}, expected {message!r}"
    for b, b0 in zip(T.bufs, before.bufs):
        assert torch.equal(b, b0), "a rejected launch wrote to its buffers"


@pytest.mark.parametrize("op", ["pcm_groupnorm_fwd", "pcm_groupnorm_bwd"])
def test_groupnorm_rejections(cuda, op):
    s = gn(op, C1=1280, C2=1312, B=1, HW=64)        # C = 2592 > kGnMaxC, a valid split into 32 groups
    T = O.materialise(s, cuda, 0)
    ws = torch.zeros(64 << 20, dtype=torch.uint8, device=cuda)     # more than any launch of it could need
    _rejected(s, T, "unsupported C", ws=ws.data_ptr(), ws_bytes=ws.numel())
    s = gn(op, C1=324, C2=316, B=1, HW=64, G=32)     # C1 % 8 != 0
    _rejected(s, O.materialise(s, cuda, 0), "bad channel split")
    s = gn(op, C1=320, C2=0, B=1, HW=64, G=24)       # C % G != 0
    _rejected(s, O.materialise(s, cuda, 0), "bad channel split")
    s = gn(op, C1=64, C2=0, B=1025, HW=8)            # B > kGnMaxB
    _rejected(s, O.materialise(s, cuda, 0), "batch too large")
    s = gn(op, C1=320, C2=0, B=2, HW=256)            # a workspace one byte short
    T = O.materialise(s, cuda, 0)
    need = O.gn_ws_need(2, O.gn_launch_cfg(320, 256, 2)[2], 320, 32)
    _rejected(s, T, "workspace too small", ws_bytes=need - 1)


def test_other_rejections(cuda):
    s = ln(True, 4, 1288)
    _rejected(s, O.materialise(s, cuda, 0), "layernorm: unsupported C")
    s = ln(False, 4, 1288)
    _rejected(s, O.materialise(s, cuda, 0), "layernorm: unsupported C")
    s = O.make_spec("pcm_add_bf16", a=True, b=True, n=1028, out=True)
    _rejected(s, O.materialise(s, cuda, 0), "add: n % 8 != 0")
    s = O.make_spec("pcm_conv3x3_c4", x=True, B=1, H=4, W=4, C=328, w=True, bias=True, sgn=1, round_in=1, out=True)
    _rejected(s, O.materialise(s, cuda, 0), "conv3x3_c4: C must be")


def test_report(cuda, capsys):
    with capsys.disabled():
        fam = ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items()))
        peak = ", ".join(f"{k[4:]} {v / 2 ** 30:.1f}" for k, v in sorted(PEAK.items(), key=lambda kv: -kv[1]))
        print(f"\nproduction norm / glue / optimiser classes: {len(CASES)} distinct; per configuration: {COUNTS}; "
              f"largest err / bound per family: {fam}; device memory peak per op (GiB): {peak}; "
              f"wall time {time.time() - T0:.0f} s (since the module was collected)")
