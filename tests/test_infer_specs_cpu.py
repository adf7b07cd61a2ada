"""The launch specs of the two inference paths - the VAE and the few-step sampler - and the float64 checker
of the VAE's glue kernels, on the CPU.

- tests/golden/infer_specs.json.gz holds every GEMM and op launch class of the recorded VAE encodes and
  decodes and sampler calls: re-recording must reproduce it, every `_call` entry point they make is covered
  by op_spec or explicitly out of scope, and every recorded GEMM descriptor passes the library's validation.
- The references of pcm_softmax_rows, pcm_transpose_bf16, pcm_latent_dist, pcm_vae_dec_in and pcm_image_exit
  accept the correct result and the result one fp32 ulp off before its output rounding, agree with the
  torch semantics of tests/vae_interp.py, and reject each mutation below.
"""
import ctypes
import importlib.util
import json
import os

import pytest
import torch

import gemm_spec as G
import op_spec as O
import vae_interp
from test_gemm_specs_cpu import Fake, _gemm
from test_op_specs_cpu import _fails, _fresh, write_ref

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
_GEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_infer_specs.py")
_s = importlib.util.spec_from_file_location("make_infer_specs", _GEN)
gen = importlib.util.module_from_spec(_s)
_s.loader.exec_module(gen)
VAE_OPS = ("pcm_softmax_rows", "pcm_transpose_bf16", "pcm_latent_dist", "pcm_vae_dec_in", "pcm_image_exit")


@pytest.fixture(scope="module")
def traces():
    """Each configuration's recorded launches, recorded once for the whole module."""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = gen.record_trace(name)
        return cache[name]
    return get


@pytest.fixture(scope="module")
def golden():
    return O.trace.load(gen.FIXTURE)


@pytest.mark.parametrize("name", gen.CONFIGS)
def test_fixture_is_current(traces, golden, name):
    got = json.loads(json.dumps(gen.distinct(traces(name))))
    hint = "regenerate with `python tests/golden/make_infer_specs.py` and say why the plan changed"
    for kind, key in (("gemm", G.launch_class), ("ops", O.launch_class)):
        want = golden[name][kind]
        have = {key(s) for s in want}
        new = [s for s in got[kind] if key(s) not in have]
        assert not new, f"{name}: {len(new)} {kind} launch classes no GPU case runs ({hint}); first: {json.dumps(new[0], sort_keys=True)}"
        assert got[kind] == want, f"{name}: the recorded {kind} launch classes differ from the fixture ({hint})"


@pytest.mark.parametrize("name", gen.CONFIGS)
def test_every_call_is_covered_or_out_of_scope(traces, name):
    names = {r["op"] for r in traces(name) if r["op"] not in ("gemm", "wgrad")}
    loose = names - set(O.ARGS) - O.OUT_OF_SCOPE
    assert not loose, f"{name}: _call entry points neither covered by op_spec nor out of scope: {sorted(loose)}"
    # attention, the DDIM step and the LoRA fuse have suites of their own (test_attn_*, test_sampler_gpu)
    assert {"pcm_attn_fwd", "pcm_sample_step", "pcm_lora_fuse"} <= O.OUT_OF_SCOPE


def test_the_inference_paths_reach_every_vae_op(golden):
    ops = {s["op"] for d in golden.values() for s in d["ops"]}
    assert set(VAE_OPS) <= ops, sorted(set(VAE_OPS) - ops)
    # the largest VAE launches: exactly 2^30 output elements, byte offsets past 2^31
    assert max(s["desc"]["M"] * s["desc"]["N"] for d in golden.values() for s in d["gemm"]) == 1 << 30


@pytest.fixture(scope="module")
def lib():
    from pcm_b200 import _lib
    return _lib.lib()


@pytest.mark.parametrize("name", gen.CONFIGS)
def test_every_inference_launch_passes_the_validation(lib, golden, name):
    for spec in golden[name]["gemm"]:
        assert spec["op"] == "gemm" and "pre" not in spec
        rc = lib.pcm_gemm_check(ctypes.byref(_gemm(spec)))
        assert rc == 0, f"{lib.pcm_last_error().decode()}: {json.dumps(spec['desc'], sort_keys=True)}"


# ---------------------------------------------------------------------------------------------
# the references of the VAE glue kernels
# ---------------------------------------------------------------------------------------------
def _softmax(rows=6, cols=1056, lds=1060, ldp=1064):
    return O.make_spec("pcm_softmax_rows", s=True, rows=rows, cols=cols, lds=lds, p=True, ldp=ldp)


def _transpose(batch=3, rows=70, cols=40, ldo=72):
    """The V third of a q / k / v matrix [batch * rows, 3 cols], as the VAE's mid-block attention reads it."""
    return O.make_spec("pcm_transpose_bf16", rows=rows, cols=cols, ldi=3 * cols, bsi=rows * 3 * cols, batch=batch,
                       ldo=ldo, bso=cols * ldo + 16, **{"in": [0, 2 * 2 * cols], "out": [1, 0]})


def _latent(noise=True, B=2, HW=77):
    return O.make_spec("pcm_latent_dist", h=True, B=B, HW=HW, w=True, bias=True, noise=True if noise else None,
                       scale=0.18215, mean=True, logvar=True, std=True, sample=True if noise else None)


SMALL = {
    "softmax": _softmax,
    "softmax_contiguous": lambda: _softmax(rows=4, cols=4096, lds=4096, ldp=4096),
    "transpose": _transpose,
    "transpose_contiguous": lambda: _transpose(batch=2, rows=96, cols=64, ldo=96),
    "latent_dist": _latent,
    "latent_dist_nonoise": lambda: _latent(noise=False),
    "vae_dec_in": lambda: O.make_spec("pcm_vae_dec_in", z=True, M=1000, w=True, bias=True, div=0.18215, out=True),
    "image_exit": lambda: O.make_spec("pcm_image_exit", x=True, B=2, HW=300, C=3, out=True, u8=True),
    "image_exit_u8": lambda: O.make_spec("pcm_image_exit", x=True, B=2, HW=300, C=3, out=None, u8=True),
}


@pytest.mark.parametrize("name", list(SMALL))
def test_correct_result_passes_and_one_ulp_off_passes(name):
    spec = SMALL[name]()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    O.guards(spec, Tout, Tin)
    for d in (1.0, -1.0):
        Tout = Tin.snapshot()
        write_ref(spec, Tin, Tout, perturb=d)
        O.check(spec, Tin, Tout)


@pytest.mark.parametrize("name", ["softmax", "transpose"])
def test_gutters_between_strided_rows_are_outside_the_windows(name):
    spec = SMALL[name]()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    lab, off, n = O.out_windows(spec)[0]
    Tout.bufs[lab][(off + n) // 2] = 0          # the first gutter element after the first row
    with pytest.raises(AssertionError, match="outside the output windows"):
        O.guards(spec, Tout, Tin)


def _interp(spec, T):
    """Run the tests/vae_interp.py statement of the op on T's buffers (fp32 torch, the kernel's layouts)."""
    op, a = spec["op"], spec["args"]
    if op == "pcm_transpose_bf16":
        x, out = O.transpose_views(T)
        vae_interp.transpose_bf16(x, out)
    elif op == "pcm_latent_dist":
        B, HW = a["B"], a["HW"]
        n = B * HW
        outs = [T.view(k, F32, 4 * n).view(B, 4, HW, 1) if a[k] else None for k in ("mean", "logvar", "std", "sample")]
        vae_interp.latent_dist(T.view("h", F32, 8 * n).view(B, HW, 1, 8), T.view("w", BF16, 64).view(8, 8),
                               T.view("bias", F32, 8), T.view("noise", F32, 4 * n).view(B, 4, HW, 1) if a["noise"] else None,
                               O.f32(a["scale"]), *outs)
    elif op == "pcm_vae_dec_in":
        M = a["M"]
        vae_interp.vae_dec_in(T.view("z", F32, 4 * M).view(M, 4), T.view("w", BF16, 16).view(4, 4),
                              T.view("bias", F32, 4), O.f32(a["div"]), T.view("out", BF16, 8 * M).view(M, 8))
    elif op == "pcm_image_exit":
        B, HW, C = a["B"], a["HW"], a["C"]
        n = B * HW * C
        vae_interp.image_exit(T.view("x", F32, n).view(B, HW, 1, C),
                              T.view("out", F32, n).view(B, C, HW, 1) if a["out"] else None,
                              T.view("u8", torch.uint8, n).view(B, HW, 1, C) if a["u8"] else None)
    else:
        raise KeyError(op)


@pytest.mark.parametrize("name", ["transpose", "latent_dist", "latent_dist_nonoise", "vae_dec_in", "image_exit",
                                  "image_exit_u8"])
def test_vae_interp_passes_the_checker(name):
    """tests/vae_interp.py (the torch statements the VAE's CPU tests run) passes the float64 checker."""
    spec = SMALL[name]()
    Tin, Tout = _fresh(spec)
    _interp(spec, Tout)
    O.check(spec, Tin, Tout)
    O.guards(spec, Tout, Tin)


def test_softmax_reference_is_the_softmax():
    spec = _softmax()
    Tin, Tout = _fresh(spec)
    s = O.softmax_scores(Tin)
    assert float(s[-1].min()) > 60           # the shifted row: exp without the max subtraction overflows fp32
    assert torch.isinf(s[-1].exp()).any()
    ref = torch.cat([p.ref for p in O.reference(spec, Tin, Tout)])
    torch.testing.assert_close(ref, torch.softmax(s.double(), -1), rtol=1e-13, atol=0)


def test_softmax_depth():
    """ceil(cols / 1024) float4s per thread: 16384 columns (SDXL's 128 x 128 latents) chain 16 of them;
    the whole sum passes through 30 roundings, not cols + 8."""
    assert O.softmax_depth(16384) == 30 and O.softmax_depth(1056) == 16 and O.softmax_depth(4) == 15


# ---------------------------------------------------------------------------------------------
# mutations: each must fail the checker
# ---------------------------------------------------------------------------------------------
def _softmax_write(spec, Tin, Tout, subtract_max=True, drop=0):
    """The kernel's fp32 arithmetic in torch, optionally without the max subtraction or with the last
    `drop` columns left out of the sum."""
    a = spec["args"]
    s = O.softmax_scores(Tin)
    x = s - s.max(1, keepdim=True).values if subtract_max else s.clone()
    e = x.exp()
    inv = 1.0 / e[:, :a["cols"] - drop].sum(1, keepdim=True)
    Tout.view("p", BF16).as_strided((a["rows"], a["cols"]), (a["ldp"], 1)).copy_((e * inv).to(BF16))


def test_mutation_softmax_without_the_max_subtraction():
    spec = _softmax()
    Tin, Tout = _fresh(spec)
    _softmax_write(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    _softmax_write(spec, Tin, Tout, subtract_max=False)
    _fails(spec, Tin, Tout, "softmax: .* non-finite")


def test_mutation_softmax_drops_the_last_four_columns():
    spec = _softmax(rows=4, cols=4096, lds=4096, ldp=4096)
    Tin, Tout = _fresh(spec)
    _softmax_write(spec, Tin, Tout, drop=4)
    _fails(spec, Tin, Tout, "softmax: .* outside the bound")


def test_mutation_transpose_with_one_tile_swapped():
    spec = _transpose()
    Tin, Tout = _fresh(spec)
    write_ref(spec, Tin, Tout)
    out = O.transpose_views(Tout)[1]
    t0, t1 = out[1, :32, :32].clone(), out[1, :32, 32:64].clone()
    out[1, :32, :32], out[1, :32, 32:64] = t1, t0
    _fails(spec, Tin, Tout, "transpose: .* differ bitwise")


def _latent_write(spec, Tin, Tout, clamp=True, std_of_logvar=0.5):
    """The kernel's result (tests/vae_interp.py), then logvar unclamped or std = exp(k logvar)."""
    _interp(spec, Tout)
    a = spec["args"]
    n = a["B"] * a["HW"]
    x = Tin.view("h", F32, 8 * n).view(n, 8).to(BF16).float()
    mo = (x @ Tin.view("w", BF16, 64).view(8, 8).float().t() + Tin.view("bias", F32, 8)).to(BF16).float()
    lv = mo[:, 4:].reshape(a["B"], a["HW"], 4).permute(0, 2, 1)
    if not clamp:
        Tout.view("logvar", F32, 4 * n).view(a["B"], 4, a["HW"]).copy_(lv)
    logvar = Tout.view("logvar", F32, 4 * n)
    Tout.view("std", F32, 4 * n).copy_((std_of_logvar * logvar).exp())
    return lv


def test_mutation_latent_dist_unclamped_logvar():
    spec = _latent()
    Tin, Tout = _fresh(spec)
    lv = _latent_write(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    assert float(lv.max()) > 20 and float(lv.min()) < -30        # moments past both clamps
    _latent_write(spec, Tin, Tout, clamp=False)
    _fails(spec, Tin, Tout, "latent_dist logvar")


def test_mutation_latent_dist_std_is_exp_logvar():
    spec = _latent()
    Tin, Tout = _fresh(spec)
    _latent_write(spec, Tin, Tout, std_of_logvar=1.0)
    _fails(spec, Tin, Tout, "latent_dist std")


def test_mutation_latent_dist_sample_with_an_fma():
    """(mean + std * noise) rounded once, as an fma would: the sample is compared bit for bit."""
    spec = _latent()
    Tin, Tout = _fresh(spec)
    _interp(spec, Tout)
    n = 2 * 77 * 4
    m, sd, z = (Tout.view("mean", F32, n).double(), Tout.view("std", F32, n).double(), Tin.view("noise", F32, n).double())
    Tout.view("sample", F32, n).copy_(((m + sd * z).float() * O.f32(0.18215)))
    _fails(spec, Tin, Tout, "latent_dist sample: .* differ bitwise")


def test_mutation_vae_dec_in_leaves_channels_4_to_7_unwritten():
    spec = SMALL["vae_dec_in"]()
    Tin, Tout = _fresh(spec)
    _interp(spec, Tout)
    O.check(spec, Tin, Tout)
    Tout.view("out", torch.int16, 8000).view(1000, 8)[:, 4:] = O.POISON
    _fails(spec, Tin, Tout, "vae_dec_in zeros: .* differ bitwise")


def test_mutation_vae_dec_in_without_the_division():
    spec = SMALL["vae_dec_in"]()
    Tin, Tout = _fresh(spec)
    _interp(dict(spec, args=dict(spec["args"], div=1.0)), Tout)
    _fails(spec, Tin, Tout, "vae_dec_in: .* outside the bound")


def _image_write(spec, Tin, Tout, rnd=torch.round, nhwc=False):
    a = spec["args"]
    n = a["B"] * a["HW"] * a["C"]
    v = (Tin.view("x", F32, n) / 2 + 0.5).clamp(0, 1)
    if a["out"]:
        out = v if nhwc else v.view(a["B"], a["HW"], a["C"]).permute(0, 2, 1).reshape(-1)
        Tout.view("out", F32, n).copy_(out)
    if a["u8"]:
        Tout.view("u8", torch.uint8, n).copy_(rnd(v * 255).to(torch.uint8))


def test_mutation_image_exit_truncates():
    spec = SMALL["image_exit"]()
    Tin, Tout = _fresh(spec)
    _image_write(spec, Tin, Tout)
    O.check(spec, Tin, Tout)
    _image_write(spec, Tin, Tout, rnd=torch.trunc)
    _fails(spec, Tin, Tout, "image_exit u8: .* differ bitwise")


def test_mutation_image_exit_rounds_half_away_from_zero():
    spec = SMALL["image_exit_u8"]()
    Tin, Tout = _fresh(spec)
    assert len(O.image_exit_ties()) > 100
    _image_write(spec, Tin, Tout, rnd=lambda y: torch.floor(y + 0.5))
    _fails(spec, Tin, Tout, "image_exit u8: .* differ bitwise")


def test_mutation_image_exit_writes_nhwc_into_the_nchw_output():
    spec = SMALL["image_exit"]()
    Tin, Tout = _fresh(spec)
    _image_write(spec, Tin, Tout, nhwc=True)
    _fails(spec, Tin, Tout, "image_exit f32: .* differ bitwise")
