"""The normalisation / glue / optimiser launch specs and their float64 checker, on the CPU.

- tests/golden/op_specs.json.gz holds every launch class of the recorded steps: re-recording must
  reproduce it (a changed launch plan fails here until the fixture, and the GPU suite, hold it), every
  `_call` entry point of the step is covered or explicitly out of scope, and every GroupNorm launch runs
  on the main stream (all of them share one workspace of self-resetting counters).
- The float64 reference agrees with the torch semantics of tests/ops_interp.py.
- The bounds catch subtle bugs: each mutation below, written into the output buffers in place of a
  correct result, fails `op_spec.check`, while the correct result perturbed by one fp32 ulp before its
  output rounding passes.
"""
import importlib.util
import json
import math
import os

import pytest
import torch

import op_spec as O
import ops_interp

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
_GEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_op_specs.py")
_s = importlib.util.spec_from_file_location("make_op_specs", _GEN)
gen = importlib.util.module_from_spec(_s)
_s.loader.exec_module(gen)


@pytest.fixture(scope="module")
def traces():
    """Each configuration's recorded step, recorded once for the whole module."""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = gen.record_trace(name)
        return cache[name]
    return get


@pytest.fixture(scope="module")
def golden():
    return O.trace.load(gen.FIXTURE)


@pytest.mark.parametrize("name", list(gen.CONFIGS))
def test_fixture_is_current(traces, golden, name):
    got = json.loads(json.dumps(O.distinct_specs(traces(name))))
    want = golden[name]
    have = {O.launch_class(s) for s in want}
    new = [s for s in got if O.launch_class(s) not in have]
    hint = "regenerate with `python tests/golden/make_op_specs.py` and say why the plan changed"
    assert not new, f"{name}: {len(new)} launch classes no GPU case runs ({hint}); first: {json.dumps(new[0], sort_keys=True)}"
    assert got == want, f"{name}: the recorded launch classes differ from the fixture ({hint})"


def test_every_call_is_covered_or_out_of_scope(traces):
    names = {r["op"] for r in traces("SD15_bs8") if r["op"] not in ("gemm", "wgrad") and not r["op"].startswith("reducer.")}
    loose = names - set(O.ARGS) - O.OUT_OF_SCOPE
    assert not loose, f"_call entry points neither covered by op_spec nor out of scope: {sorted(loose)}"
    assert not set(O.ARGS) & O.OUT_OF_SCOPE
    from pcm_b200 import _lib
    assert set(O.ARGS) | O.OUT_OF_SCOPE <= set(_lib.EXPORTS)


@pytest.mark.parametrize("name", list(gen.CONFIGS))
def test_groupnorm_stays_on_the_main_stream(traces, name):
    side = [r for r in traces(name) if r["op"] in O.GN_OPS and r["side"]]
    assert not side, f"{name}: {len(side)} GroupNorm launches on the weight-gradient stream would race on the shared counters"


def test_fixture_covers_every_op(golden):
    """The training steps' fixture and the inference paths' (tests/golden/infer_specs.json.gz: the VAE's
    glue kernels) together launch every covered op."""
    infer = O.trace.load(os.path.join(os.path.dirname(gen.FIXTURE), "infer_specs.json.gz"))
    ops = {s["op"] for specs in golden.values() for s in specs} | {s["op"] for d in infer.values() for s in d["ops"]}
    assert ops == set(O.ARGS), sorted(set(O.ARGS) - ops)


def test_workspace_restatement():
    """gn_ws_bytes mirrors pcm_groupnorm_ws_bytes (the GPU suite asserts equality with the library):
    the one-image partition bounds every batch's, and the merge fits kGnStage."""
    for C, HW in ((320, 4096), (320, 16384), (2560, 64), (96, 100), (640, 1024)):
        cfg1 = O.gn_launch_cfg(C, HW, 1)
        for B in (1, 2, 6, 8, 24):
            threads, ppb, nblk = O.gn_launch_cfg(C, HW, B)
            assert nblk <= cfg1[2] and nblk * 32 <= O.GN_STAGE and threads >= 8 * 32
            assert O.gn_ws_need(B, nblk, C, 32) <= O.gn_ws_bytes(B, HW, C, 32)
    assert O.gn_launch_cfg(320, 16384, 2)[2] * 32 == O.GN_STAGE     # SDXL's block cap fills the stage exactly


# ---------------------------------------------------------------------------------------------
# writing results into the output windows
# ---------------------------------------------------------------------------------------------
def write_ref(spec, Tin, Tout, perturb=0.0):
    """Write the reference into Tout's outputs (rounded to each output's dtype), optionally perturbed by
    `perturb` fp32 ulps before the rounding (where the bound allows any error: an element bounded by zero, a
    logvar past its clamp, is exact).  Pieces are written in order, so later pieces (GroupNorm's output,
    computed on the written statistics) see the earlier ones."""
    for p in O.reference(spec, Tin, Tout):
        ref = p.ref.reshape(p.got.shape)
        if p.bnd is not None and perturb and ref.dtype == F64:
            off = ref.float().double() * (1 + perturb * 2.0 ** -23)
            ref = torch.where(torch.as_tensor(p.bnd).reshape(ref.shape) > 0, off, ref)
        p.got.copy_(ref.to(p.got.dtype))


def _fresh(spec, seed=0):
    T = O.materialise(spec, "cpu", seed)
    return T, T.snapshot()


def _fails(spec, Tin, Tout, match=None):
    with pytest.raises(AssertionError, match=match):
        O.check(spec, Tin, Tout)


def _gn_spec(op="pcm_groupnorm_fwd", C1=320, C2=0, B=2, HW=64, G=32, eps=1e-5, silu=1, add=True, colsum=True):
    if op == "pcm_groupnorm_bwd":
        return O.make_spec(op, dy=True, x1=True, x2=True if C2 else None, C1=C1, C2=C2, B=B, HW=HW, G=G,
                           gamma=True, beta=True, eps=eps, silu=silu, stats=True, red=True, add=True if add else None,
                           dx1=True, dx2=True if C2 else None, colsum=True if colsum else None)
    return O.make_spec(op, x1=True, x2=True if C2 else None, C1=C1, C2=C2, B=B, HW=HW, G=G, gamma=True, beta=True,
                       eps=eps, silu=silu, out=True, stats=True)


SMALL = {
    "gn_fwd": lambda: _gn_spec(C1=40, C2=56, G=32),
    "gn_bwd": lambda: _gn_spec("pcm_groupnorm_bwd", C1=40, C2=56, G=32),
    "gn_bwd_noadd": lambda: _gn_spec("pcm_groupnorm_bwd", C1=320, silu=0, add=False, colsum=False),
    "ln_fwd": lambda: O.make_spec("pcm_layernorm_fwd", x=True, M=37, C=320, gamma=True, beta=True, eps=1e-5, out=True, stats=True),
    "ln_bwd": lambda: O.make_spec("pcm_layernorm_bwd", dy=True, x=True, M=37, C=640, gamma=True, stats=True, add=True, dx=True),
    "geglu_fwd": lambda: O.make_spec("pcm_geglu_fwd", u=True, M=64, F=1280, out=True),
    "geglu_bwd": lambda: O.make_spec("pcm_geglu_bwd", dgg=True, u=True, M=64, F=1280, du=True),
    "up_fwd": lambda: O.make_spec("pcm_upsample2x_fwd", x=True, B=2, H=4, W=3, C=16, out=True),
    "up_bwd": lambda: O.make_spec("pcm_upsample2x_bwd", dout=True, B=2, H=4, W=3, C=16, din=True),
    "conv": lambda: O.make_spec("pcm_conv3x3_c4", x=True, B=2, H=5, W=6, C=16, w=True, bias=True, sgn=1, round_in=1, out=True),
    "conv_dgrad": lambda: O.make_spec("pcm_conv3x3_c4", x=True, B=2, H=5, W=6, C=16, w=True, bias=None, sgn=-1, round_in=0, out=True),
    "timestep": lambda: O.make_spec("pcm_timestep_embed", t=True, B=5, C=320, out=True),
    "add": lambda: O.make_spec("pcm_add_bf16", a=True, b=True, n=1024, out=True),
    "cast": lambda: O.make_spec("pcm_cast_f32_bf16", x=True, n=1001, out=True),
    "sumsq": lambda: O.make_spec("pcm_grad_sumsq", g=True, n=1027, out=True),
    "adamw": lambda: O.make_spec("pcm_adamw_clip", p=True, g=True, m=True, v=True, n=1003, state=True, beta1=0.9,
                                 beta2=0.999, eps=1e-8, wd=0.01, max_norm=1.0, inv_world=0.5, sumsq=True, zero_grad=1),
    "ema": lambda: O.make_spec("pcm_ema_update", targ=True, src=True, n=999, rate=0.95),
}


@pytest.mark.parametrize("name", list(SMALL))
def test_correct_result_passes_and_one_ulp_off_passes(name):
    spec = SMALL[name]()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    for d in (1.0, -1.0):
        Tout = Tin.snapshot()
        write_ref(spec, Tin, Tout, perturb=d)
        O.check(spec, Tin, Tout)


def test_refresh_reference_writes_the_four_layouts():
    table = [[0, 64 * 128, 0, 64 * 128, 64 * 128 + 256 * 64, 64 * 128 + 2 * 256 * 64, 128 | (1 << 32), 256 | (64 << 32), 0]]
    spec = O.make_spec("pcm_lora_refresh", table, master=True, table=True, num_entries=1, total_work=6,
                       scale=0.125, opnd=True)
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    A = Tin.view("master", F32)[:64 * 128].view(64, 128)
    sB = Tin.view("master", F32)[64 * 128:64 * 128 + 256 * 64].view(256, 64) * 0.125
    o = Tout.view("opnd", BF16)
    assert torch.equal(o[:64 * 128].view(64, 128), A.to(BF16))
    assert torch.equal(o[64 * 128 + 2 * 256 * 64:].view(128, 64), A.t().to(BF16))
    assert torch.equal(o[64 * 128 + 256 * 64:64 * 128 + 2 * 256 * 64].view(64, 256), sB.t().to(BF16))
    o[5] = o[5].float() * 1.0078125
    _fails(spec, Tin, Tout, "bitwise")


# ---------------------------------------------------------------------------------------------
# the reference against tests/ops_interp.py
# ---------------------------------------------------------------------------------------------
def _interp_vs_ref(spec, run, pieces_of):
    """Run the ops_interp wrapper (fp32 outputs) and compare with the float64 reference's pieces."""
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    want = run(Tin)
    got = [p.ref for p in O.reference(spec, Tin, Tout) if p.fam in pieces_of]
    got = torch.cat([g.reshape(-1) for g in got])
    torch.testing.assert_close(got.float(), want.reshape(-1).float(), rtol=2e-4, atol=2e-4)


def test_reference_agrees_with_ops_interp():
    # GroupNorm forward (x1 | x2 concat, SiLU): out in fp32
    s = _gn_spec(C1=40, C2=56, G=32, B=2, HW=16)
    a = s["args"]

    def gn(T):
        x1 = T.view("x1", BF16, 2 * 16 * 40).view(32, 40)
        x2 = T.view("x2", BF16, 2 * 16 * 56).view(32, 56)
        out, st = torch.empty(32, 96), torch.empty(2, 32, 2)
        ops_interp.groupnorm_fwd(x1, x2, T.view("gamma", F32, 96), T.view("beta", F32, 96), a["eps"], 1, out, st, 2, 16)
        return torch.cat([o.reshape(-1) for o in out.view(2, 16, 96)])
    _interp_vs_ref(s, gn, {"gn fwd"})

    # GroupNorm backward (SiLU, add, colsum) on the reference's own statistics
    s = _gn_spec("pcm_groupnorm_bwd", C1=320, B=2, HW=16)

    def gnb(T):
        x1 = T.view("x1", BF16, 32 * 320).view(32, 320)
        dx1, cs = torch.empty(32, 320), torch.empty(2, 320)
        ops_interp.groupnorm_bwd(T.view("dy", BF16, 32 * 320).view(32, 320), x1, None, T.view("gamma", F32, 320),
                                 T.view("beta", F32, 320), 1e-5, 1, None, None, T.view("add", BF16, 32 * 320).view(32, 320),
                                 dx1, None, 2, 16, colsum=cs)
        return dx1
    _interp_vs_ref(s, gnb, {"gn bwd"})

    s = SMALL["ln_fwd"]()

    def ln(T):
        out, st = torch.empty(37, 320), torch.empty(37, 2)
        ops_interp.layernorm_fwd(T.view("x", BF16, 37 * 320).view(37, 320), T.view("gamma", F32, 320),
                                 T.view("beta", F32, 320), out, st)
        return out
    _interp_vs_ref(s, ln, {"ln fwd"})

    s = O.make_spec("pcm_layernorm_bwd", dy=True, x=True, M=37, C=640, gamma=True, stats=True, add=True, dx=True)

    def lnb(T):
        dx = torch.empty(37, 640)
        ops_interp.layernorm_bwd(T.view("dy", BF16, 37 * 640).view(37, 640), T.view("x", BF16, 37 * 640).view(37, 640),
                                 T.view("gamma", F32, 640), None, T.view("add", BF16, 37 * 640).view(37, 640), dx)
        return dx
    _interp_vs_ref(s, lnb, {"ln bwd"})

    s = SMALL["geglu_bwd"]()

    def gb(T):
        du = torch.empty(64, 2560)
        ops_interp.geglu_bwd(T.view("dgg", BF16, 64 * 1280).view(64, 1280), T.view("u", BF16, 64 * 2560).view(64, 2560), du)
        return du.view(64, 2, 1280).permute(1, 0, 2)
    _interp_vs_ref(s, gb, {"geglu bwd"})

    s = SMALL["geglu_fwd"]()

    def gf(T):
        out = torch.empty(64, 1280)
        ops_interp.geglu_fwd(T.view("u", BF16, 64 * 2560).view(64, 2560), out)
        return out
    _interp_vs_ref(s, gf, {"geglu fwd"})

    for name in ("conv", "conv_dgrad"):
        s = SMALL[name]()
        a = s["args"]

        def cv(T, a=a):
            out = torch.empty(2, 5, 6, 16)
            ops_interp.conv3x3_c4(T.view("x", F32, 2 * 5 * 6 * 4).view(2, 5, 6, 4), T.view("w", BF16, 36 * 16).view(16, 3, 3, 4),
                                  T.view("bias", F32, 16) if a["bias"] else None, out, a["sgn"], bool(a["round_in"]))
            return out
        _interp_vs_ref(s, cv, {"conv_c4"})

    s = SMALL["timestep"]()

    def ts(T):
        out = torch.empty(5, 320)
        ops_interp.timestep_embed(T.view("t", torch.int64, 5), out)
        return out
    _interp_vs_ref(s, ts, {"timestep"})


def test_optimiser_reference_agrees_with_ops_interp():
    s = SMALL["adamw"]()
    Tin, Tout = _fresh(s)
    write_ref(s, Tin, Tout)
    T2 = Tin.snapshot()                  # the fp32 torch update of ops_interp passes the float64 check
    calls = ops_interp.PcmCalls()        # (given the float arguments as the kernel receives them, in fp32)
    calls.pcm_adamw_clip(*(T2.addr(k) if isinstance(v, list) else O.f32(v) if isinstance(v, float) else v
                           for k, v in s["args"].items()))
    O.check(s, Tin, T2)
    s = SMALL["sumsq"]()
    Tin, Tout = _fresh(s)
    write_ref(s, Tin, Tout)
    calls.pcm_grad_sumsq(Tin.addr("g"), 1027, Tin.addr("out"))
    assert math.isclose(float(Tin.view("out", F64, 1)), float(Tout.view("out", F64, 1)), rel_tol=1e-12)


# ---------------------------------------------------------------------------------------------
# mutations: each must fail the checker
# ---------------------------------------------------------------------------------------------
def _gn_write(spec, Tin, Tout, stats_fn, chan_map=None):
    """A GroupNorm forward result from given float64 statistics: stats [B, G, 2] written as fp32, the output
    from them in float64, rounded once; chan_map[c] = the group channel c takes its statistics from."""
    a = spec["args"]
    B, HW, G, C1, C2 = a["B"], a["HW"], a["G"], a["C1"], a["C2"]
    C = C1 + C2
    st = stats_fn(Tin)
    Tout.view("stats", F32, 2 * B * G).copy_(st.reshape(-1).float())
    gmap = torch.arange(C) // (C // G) if chan_map is None else chan_map
    gamma, beta = Tin.view("gamma", F32, C).double(), Tin.view("beta", F32, C).double()
    out = Tout.view("out", BF16, B * HW * C).view(B, HW, C)
    for b in range(B):
        X = O.gn_image(Tin, b)
        y = (X - st[b, gmap, 0].float().double()) * st[b, gmap, 1].float().double() * gamma + beta
        out[b].copy_((O._silu(y) if a["silu"] else y).to(BF16))


def test_mutation_groupnorm_unbiased_variance():
    spec = _gn_spec(C1=320, B=2, HW=64)
    Tin, Tout = _fresh(spec)
    a = spec["args"]

    def unbiased(T):
        st = []
        for b in range(2):
            Xg = O.gn_image(T, b).view(64, 32, 10)
            st.append(torch.stack([Xg.mean((0, 2)), (Xg.reshape(-1, 32, 10).permute(1, 0, 2).reshape(32, -1).var(1)
                                                     + O.f32(a["eps"])).rsqrt()], 1))
        return torch.stack(st)
    _gn_write(spec, Tin, Tout, lambda T: O.gn_stats64(T, a["eps"]))
    O.check(spec, Tin, Tout)
    _gn_write(spec, Tin, Tout, unbiased)
    _fails(spec, Tin, Tout, "gn stats")


def test_mutation_groupnorm_straddle_channel_uses_the_wrong_group():
    spec = _gn_spec(C1=40, C2=56, G=32)          # cpg 3: group 13 = channels 39 | 40, 41 straddles x1 / x2
    Tin, Tout = _fresh(spec)
    eps = spec["args"]["eps"]
    cmap = torch.arange(96) // 3
    _gn_write(spec, Tin, Tout, lambda T: O.gn_stats64(T, eps), cmap)
    O.check(spec, Tin, Tout)
    cmap[40] = 14
    _gn_write(spec, Tin, Tout, lambda T: O.gn_stats64(T, eps), cmap)
    _fails(spec, Tin, Tout, "gn fwd")


def test_mutation_groupnorm_wrong_eps_on_a_near_eps_group():
    spec = _gn_spec(C1=320, B=1, HW=64, eps=1e-6, silu=0)
    Tin, Tout = _fresh(spec)
    x = Tin.view("x1", BF16, 64 * 320).view(64, 320)
    g = torch.Generator().manual_seed(3)
    x[:, :10] = (torch.randn(64, 10, generator=g) * 1e-3).to(BF16)    # group 0: variance 1e-6, near eps
    Tout = Tin.snapshot()
    _gn_write(spec, Tin, Tout, lambda T: O.gn_stats64(T, 1e-6))
    O.check(spec, Tin, Tout)
    _gn_write(spec, Tin, Tout, lambda T: O.gn_stats64(T, 1e-5))
    _fails(spec, Tin, Tout, "gn stats")
    # the unit-variance groups alone would not show it
    d = (O.gn_stats64(Tin, 1e-5) - O.gn_stats64(Tin, 1e-6))[0, 1:, 1] / O.gn_stats64(Tin, 1e-6)[0, 1:, 1]
    assert float(d.abs().max()) < 2 ** -8


def test_mutation_layernorm_backward_without_the_xhat_term():
    spec = SMALL["ln_bwd"]()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    M, C = 37, 640
    X = Tin.view("x", BF16, M * C).view(M, C).double()
    st = Tin.view("stats", F32, 2 * M).view(M, 2).double()
    g = Tin.view("dy", BF16, M * C).view(M, C).double() * Tin.view("gamma", F32, C).double()
    dx = st[:, 1:] * (g - g.mean(1, keepdim=True)) + Tin.view("add", BF16, M * C).view(M, C).double()
    Tout.view("dx", BF16, M * C).copy_(dx.reshape(-1).to(BF16))
    _fails(spec, Tin, Tout, "ln bwd")


def _tanh_gelu(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def _dtanh_gelu(x):
    k = math.sqrt(2 / math.pi)
    t = torch.tanh(k * (x + 0.044715 * x ** 3))
    return 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * k * (1 + 3 * 0.044715 * x * x)


def test_mutation_tanh_gelu_forward():
    spec = O.make_spec("pcm_geglu_fwd", u=True, M=512, F=1280, out=True)
    Tin, Tout = _fresh(spec)
    u = Tin.view("u", BF16, 512 * 2560).view(512, 2560).double()
    Tout.view("out", BF16, 512 * 1280).copy_((u[:, :1280] * _tanh_gelu(u[:, 1280:])).reshape(-1).to(BF16))
    _fails(spec, Tin, Tout, "outside the bound|signed error")


def test_mutation_tanh_gelu_backward():
    spec = O.make_spec("pcm_geglu_bwd", dgg=True, u=True, M=512, F=1280, du=True)
    Tin, Tout = _fresh(spec)
    u = Tin.view("u", BF16, 512 * 2560).view(512, 2560).double()
    d = Tin.view("dgg", BF16, 512 * 1280).view(512, 1280).double()
    x, g = u[:, :1280], u[:, 1280:]
    du = torch.cat([d * _tanh_gelu(g), d * x * _dtanh_gelu(g)], 1)
    Tout.view("du", BF16, 512 * 2560).copy_(du.reshape(-1).to(BF16))
    _fails(spec, Tin, Tout, "outside the bound|signed error")


def test_mutation_upsample_backward_in_another_order():
    spec = SMALL["up_bwd"]()
    Tin, Tout = _fresh(spec)
    d = Tin.view("dout", BF16, 2 * 8 * 6 * 16).view(2, 8, 6, 16)
    # taps 1, 3 2^-26, 3 2^-26, -1: the kernel's order rounds both small taps away (0); starting from -1 keeps them
    d[0, 0, 0, 0], d[0, 0, 1, 0], d[0, 1, 0, 0], d[0, 1, 1, 0] = 1.0, 3 * 2.0 ** -26, 3 * 2.0 ** -26, -1.0
    Tout = Tin.snapshot()
    write_ref(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    v = d.view(2, 4, 2, 3, 2, 16).float()
    s = ((v[:, :, 1, :, 1] + v[:, :, 0, :, 1]) + v[:, :, 1, :, 0]) + v[:, :, 0, :, 0]
    assert float(s[0, 0, 0, 0]) == 2.0 ** -23
    Tout.view("din", BF16, 2 * 4 * 3 * 16).copy_(s.to(BF16).reshape(-1))
    _fails(spec, Tin, Tout, "bitwise")


def test_mutation_conv_c4_taps_not_flipped():
    spec = SMALL["conv_dgrad"]()
    Tin, Tout = _fresh(spec)
    wrong = dict(spec, args=dict(spec["args"], sgn=1))
    write_ref(wrong, Tin, Tout)
    _fails(spec, Tin, Tout, "conv_c4")


def test_mutation_sumsq_without_the_tail():
    spec = SMALL["sumsq"]()                      # n = 4 * 256 + 3
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    Tout.view("out", F64, 1)[0] = Tin.view("g", F32, 1024).double().square().sum()
    _fails(spec, Tin, Tout, "sumsq")


def _adamw_write(spec, Tin, Tout, bias_correction=True, clip_before_fold=False, step=None):
    a = spec["args"]
    n = a["n"]
    b1, b2, eps, wd, mx, iw = (O.f32(a[k]) for k in ("beta1", "beta2", "eps", "wd", "max_norm", "inv_world"))
    st = Tin.view("state", F32, 2).double()
    lr, k = float(st[0]), float(st[1]) + 1 if step is None else step
    norm = math.sqrt(float(Tin.view("sumsq", F64, 1)[0])) * (1.0 if clip_before_fold else iw)
    coef = min(mx / (norm + 1e-6), 1.0) * iw
    p, g = Tin.view("p", F32, n).double(), Tin.view("g", F32, n).double() * coef
    m = b1 * Tin.view("m", F32, n).double() + (1 - b1) * g
    v = b2 * Tin.view("v", F32, n).double() + (1 - b2) * g * g
    bc1, bc2 = (1 - b1 ** k, 1 - b2 ** k) if bias_correction else (1.0, 1.0)
    p = p * (1 - lr * wd) - lr / bc1 * m / (v.sqrt() / math.sqrt(bc2) + eps)
    for name, val in (("p", p), ("m", m), ("v", v)):
        Tout.view(name, F32, n).copy_(val.float())
    Tout.view("state", F32, 2).copy_(torch.tensor([lr, float(st[1]) + 1]))
    Tout.view("g", F32, n).zero_()


def test_mutation_adamw_without_bias_correction():
    spec = SMALL["adamw"]()
    Tin, Tout = _fresh(spec)
    _adamw_write(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    _adamw_write(spec, Tin, Tout, bias_correction=False)
    _fails(spec, Tin, Tout, "adamw")


def test_mutation_adamw_clip_before_the_world_fold():
    spec = SMALL["adamw"]()                      # inv_world = 1/2, the clip active
    Tin, Tout = _fresh(spec)
    Tin.view("g", F32, 1003).mul_(100)
    Tin.view("sumsq", F64, 1)[0] = Tin.view("g", F32, 1003).double().square().sum() * 4     # the summed gradient of 2 ranks
    Tout = Tin.snapshot()
    _adamw_write(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    _adamw_write(spec, Tin, Tout, clip_before_fold=True)
    _fails(spec, Tin, Tout, "adamw")


def test_mutation_adamw_second_update_with_step_one():
    spec = SMALL["adamw"]()
    T0, T1 = _fresh(spec)
    write_ref(spec, T0, T1)                      # update 1 (state step 0 -> 1)
    T2 = T1.snapshot()
    _adamw_write(spec, T1, T2)                   # update 2 from the device-side state
    O.check(spec, T1, T2)
    _adamw_write(spec, T1, T2, step=1.0)
    _fails(spec, T1, T2, "adamw")


@pytest.mark.parametrize("name", ["add", "cast", "geglu_fwd", "ln_fwd", "gn_bwd", "conv", "ema", "adamw"])
def test_mutation_grid_stride_loop_skips_its_last_stride(name):
    spec = SMALL[name]()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    lab, off, n = O.out_windows(spec)[0]
    w = Tout.bufs[lab][off // 2:(off + n) // 2]
    w[-max(8, w.numel() // 7):] = O.POISON          # the last stride of a 7-stride loop never ran
    _fails(spec, Tin, Tout, "non-finite|bitwise")


@pytest.mark.parametrize("name", ["add", "sumsq", "adamw", "ema"])
def test_sliced_references(monkeypatch, name):
    """The flat optimiser / add references run in slices of op_spec.SLICE elements (the GPU holds them in
    float64 one slice at a time); with slices of 100 a correct result passes and a wrong last element fails."""
    monkeypatch.setattr(O, "SLICE", 100)
    spec = SMALL[name]()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    assert len([p for p in O.reference(spec, Tin, Tout) if p.fam.split()[0] in ("add_bf16", "adamw", "ema")]) \
        >= (0 if name == "sumsq" else 10)
    O.check(spec, Tin, Tout)
    if name == "sumsq":
        Tout.view("out", F64, 1)[0] *= 1 + 2.0 ** -20
    else:                       # the last element of the first output, in the last slice: its top 16 bits + 1
        lab, off, n = O.out_windows(spec)[0]
        Tout.bufs[lab][(off + n) // 2 - 1] += 1
    _fails(spec, Tin, Tout)
