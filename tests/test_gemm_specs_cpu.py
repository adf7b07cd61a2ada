"""The GEMM launch specs, their float64 oracle and the descriptor validation, without a GPU.

* The fixture tests/golden/gemm_specs.json.gz must equal a fresh dry run of every configuration, so a change
  to the launch plan fails here until the GPU suite (test_gemm_prod_gpu.py) holds the new launch.
* gemm_spec.reference is pinned against F.linear / F.conv2d / autograd in float64 on hand-built launches and
  against the independently written interpreter tests/gemm_interp.py on the recorded TINY step.
* gemm_spec.check has teeth: references corrupted the way a kernel bug would corrupt the output are rejected.
* pcm_gemm / pcm_wgrad reject descriptors the kernels cannot serve with an error naming the field, and accept
  every recorded production launch.  Only pcm_gemm_check / pcm_wgrad_check are called, which run the host
  checks and launch nothing; that the launch functions run the same checks first is read from the source.

A change that alters the plan on purpose regenerates the fixture with
`python tests/golden/make_gemm_specs.py` and says in its description why the plan changed."""
import copy
import ctypes
import importlib.util
import json
import os

import pytest
import torch
import torch.nn.functional as F

import gemm_interp
import gemm_spec as G
import test_gemm_gpu as old_suite
from gemm_cases import (concat_lora_spec, conv3x3_spec, dgrad2_spec, grouped_spec, linear_spec, stride2_spec,
                        wgrad_spec)

_GEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_gemm_specs.py")
_s = importlib.util.spec_from_file_location("make_gemm_specs", _GEN)
gen = importlib.util.module_from_spec(_s)
_s.loader.exec_module(gen)

BF16 = torch.bfloat16
CPU = torch.device("cpu")


@pytest.fixture(scope="module")
def golden():
    return G.trace.load(gen.FIXTURE)


@pytest.mark.parametrize("name", list(gen.CONFIGS))
def test_fixture_is_current(golden, name):
    got = json.loads(json.dumps(gen.record(name)))
    want = golden[name]
    have = {G.launch_class(s) for s in want}
    new = [s for s in got if G.launch_class(s) not in have]
    hint = "regenerate with `python tests/golden/make_gemm_specs.py` and say why the plan changed"
    assert not new, f"{name}: {len(new)} launch classes no GPU case runs ({hint}); first: {json.dumps(new[0], sort_keys=True)}"
    assert got == want, f"{name}: the recorded launch classes differ from the fixture ({hint})"


def _nchw(T, a):
    return T.asrc(a, 0).double().permute(0, 3, 1, 2)


def _w4(T, b, Cin):
    """[Cout, (kh, kw, Cin)] tap-major weights -> [Cout, Cin, 3, 3]."""
    return T.bsrc(b).double().reshape(b["N"], 3, 3, Cin).permute(0, 3, 1, 2)


def _agree(ref, want):
    torch.testing.assert_close(ref, want, rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------
# the oracle against torch
# ---------------------------------------------------------------------------------------------
def test_reference_conv3x3_matches_conv2d():
    spec = conv3x3_spec(B=3, H=4, W=8, act=1)
    T, d = G.materialise(spec, CPU), spec["desc"]
    ref, S, base = G.reference(spec, T)
    want = F.conv2d(_nchw(T, d["a"][0]), _w4(T, d["b"][0], 64), T.flat(d["bias"], torch.float32)[:96].double(), padding=1)
    _agree(ref, F.silu(want).permute(0, 2, 3, 1).reshape(-1, 96))
    assert (base.double() - ref).abs().max() < 1e-4


def test_reference_s_is_the_sum_of_absolute_values():
    """S, on which the bound rests, against an independent computation: the same convolution of |x| with |w|."""
    spec = conv3x3_spec(B=3, H=4, W=8, rowvec=True, residual=True, alpha=0.5)
    T, d = G.materialise(spec, CPU), spec["desc"]
    ref, S, _ = G.reference(spec, T)
    want = 0.5 * F.conv2d(_nchw(T, d["a"][0]).abs(), _w4(T, d["b"][0], 64).abs(), padding=1).permute(0, 2, 3, 1)
    want = want + T.flat(d["bias"], torch.float32)[:96].double().abs()
    want = want + T.flat(d["rowvec"], BF16).as_strided((3, 96), (d["rowvec_ld"], 1)).double().abs()[:, None, None, :]
    want = want.reshape(-1, 96) + T.flat(d["residual"], BF16)[T.out_index(d)].double().abs()
    _agree(S, want)
    assert (S >= ref.abs()).all()


def test_reference_stride2_dgrad_matches_autograd():
    """The four parity-plane launches together are conv2d's input gradient, each stored only into its plane."""
    B, H, W = 2, 8, 8
    dx = torch.zeros(B, H, W, 64, dtype=torch.float64)
    g = torch.Generator().manual_seed(0)
    dy = torch.randn(B, H // 2, W // 2, 64, generator=g).to(BF16)
    wt = (torch.randn(64, 9 * 64, generator=g) / 24).to(BF16)          # [Cin, (tap, Cout)]
    for p in range(2):
        for q in range(2):
            spec = dgrad2_spec(p, q, B=B, H=H, W=W)
            T, d = G.materialise(spec, CPU), spec["desc"]
            T.asrc(d["a"][0], 0).copy_(dy)
            T.bsrc_view(d["b"][0]).copy_(wt)
            dx[:, p::2, q::2] = G.reference(spec, T)[0].view(B, H // 2, W // 2, 64)
            idx = T.out_index(d).view(B, H // 2, W // 2, 64)
            assert (idx[0, 0, 1, 0] - idx[0, 0, 0, 0], idx[0, 1, 0, 0] - idx[0, 0, 0, 0]) == (2 * 72, 2 * W * 72)
    x = torch.zeros(B, 64, H, W, dtype=torch.float64, requires_grad=True)
    w4 = wt.double().view(64, 3, 3, 64).permute(3, 0, 1, 2)             # [Cout, Cin, kh, kw]
    F.conv2d(x, w4, stride=2, padding=1).backward(dy.double().permute(0, 3, 1, 2))
    _agree(dx, x.grad.permute(0, 2, 3, 1))


def test_reference_stride2_matches_conv2d():
    spec = stride2_spec()
    T, d = G.materialise(spec, CPU), spec["desc"]
    # the four planes are views of one image: plane (0, 0) starts it
    x = T.flat(d["a"][0]["ptr"], BF16)[:2 * 8 * 8 * 64].view(2, 8, 8, 64).double().permute(0, 3, 1, 2)
    want = F.conv2d(x, _w4(T, d["b"][0], 64), stride=2, padding=1)
    _agree(G.reference(spec, T)[0], want.permute(0, 2, 3, 1).reshape(-1, 64))


def test_reference_concat_lora_matches_conv2d():
    spec = concat_lora_spec()
    T, d = G.materialise(spec, CPU), spec["desc"]
    w = T.bsrc(d["b"][0]).double()
    w1 = w[:, :9 * 128].reshape(96, 3, 3, 128).permute(0, 3, 1, 2)
    w2 = w[:, 9 * 128:].reshape(96, 3, 3, 64).permute(0, 3, 1, 2)
    want = F.conv2d(_nchw(T, d["a"][0]), w1, padding=1) + F.conv2d(_nchw(T, d["a"][1]), w2, padding=1)
    want = want.permute(0, 2, 3, 1).reshape(-1, 96) + T.asrc(d["a"][2], 0).double().reshape(-1, 24) @ T.bsrc(d["b"][1]).double().t()
    _agree(G.reference(spec, T)[0], want)


def test_reference_grouped_n_ranges_matches_linear():
    spec = grouped_spec()
    T, d = G.materialise(spec, CPU), spec["desc"]
    x, t = T.asrc(d["a"][0], 1)[0, 0].double(), T.asrc(d["a"][1], 1)[0, 0].double()
    want = F.linear(x, T.bsrc(d["b"][0]).double())
    sb = T.bsrc(d["b"][1]).double()
    for i in range(3):
        want[:128, 64 * i:64 * i + 64] += t[:, 64 * i:64 * i + 64] @ sb[64 * i:64 * i + 64].t()
    want += T.flat(d["residual"], BF16)[T.out_index(d)].double()
    _agree(G.reference(spec, T)[0], want)


@pytest.mark.parametrize("lin", [True, False])
def test_reference_wgrad_matches_autograd(lin):
    spec = wgrad_spec(lin, qC=128, q_c0=64)
    T, d = G.materialise(spec, CPU), spec["desc"]
    out0 = T.flat(d["out"], torch.float32)[T.wgrad_index(d)].double()
    ref = G.reference_wgrad(spec, T)[0]
    if lin:
        p, q = T.asrc(d["p"], 1)[0, 0].double(), T.asrc(d["q"], 1)[0, 0].double()[:, 64:]
        a = torch.zeros(64, 96, dtype=torch.float64, requires_grad=True)
        F.linear(p, a).backward(q)
        want = a.grad.t()[None]
    else:
        a = torch.zeros(64, 96, 3, 3, dtype=torch.float64, requires_grad=True)
        F.conv2d(_nchw(T, d["p"]), a, padding=1).backward(_nchw(T, d["q"])[:, 64:])
        want = a.grad.permute(2, 3, 1, 0).reshape(9, 96, 64)
    _agree(ref, want * d["alpha"] + out0)


def test_reference_agrees_with_gemm_interp_on_the_tiny_step():
    """Two independently written statements of the descriptor semantics, on every launch class of TINY."""
    from pcm_b200 import _lib
    specs = G.distinct_specs(G.trace.record("TINY", {}))
    n = 0
    for spec in specs:
        if spec["op"] != "gemm":
            continue
        spec = {k: v for k, v in spec.items() if k != "pre"}
        T, d = G.materialise(spec, CPU, seed=n), spec["desc"]
        if "pre" not in spec and d["dep_a_src1"]:       # the producer is not run here: T holds real values
            G._fill(T.asrc(d["a"][d["dep_a_src1"] - 1], d["lin"]), torch.Generator().manual_seed(n))
        ref = G.reference(spec, T)[0]
        s = G.gemm_desc(d, T)
        res = None
        if d["residual"]:
            res = T.flat(d["residual"], BF16)[T.out_index(d)].clone()
        nb = (d["M"] - 1) // d["epiHW"] + 1
        rv = T.flat(d["rowvec"], BF16).as_strided((nb, d["N"]), (d["rowvec_ld"], 1)) if d["rowvec"] else None
        out = torch.empty(d["M"], d["N"], dtype=torch.float64)
        prog = [(e["a_src"], e["b_src"], e["dw"], e["dh"], e["nchunks"], e["a_c0"], e["b_k0"], e["n_lo"], e["n_hi"]) for e in d["prog"]]
        got = gemm_interp.interp_gemm(list(s.a)[:d["num_a"]], list(s.b)[:d["num_b"]], prog, lin=d["lin"], M=d["M"], N=d["N"],
                                      out=out.float(), geo=(d["geoW"], d["geoH"]),
                                      bias=T.flat(d["bias"], torch.float32) if d["bias"] else None, residual=res,
                                      act=d["act"], rowvec=rv, alpha=d["alpha"])
        torch.testing.assert_close(got.double(), ref, rtol=1e-4, atol=1e-4)
        n += 1
    assert n > 20


# ---------------------------------------------------------------------------------------------
# the comparator has teeth
# ---------------------------------------------------------------------------------------------
def _rounded(x, d):
    return x.to(torch.float32 if (d["out_fp32"] and not d["round_bf16"]) else BF16).double()


def _drop_last16(spec, T):
    e = spec["desc"]["prog"][4]
    b = spec["desc"]["b"][e["b_src"]]
    T.bsrc(b)[:, e["b_k0"] + 64 * e["nchunks"] - 16:e["b_k0"] + 64 * e["nchunks"]] = 0


def _corrupt_desc(edit):
    def f(spec, T):
        d = copy.deepcopy(spec["desc"])
        edit(d)
        return G.reference(spec, T, desc=d)[0]
    return f


def _corrupt_tensors(edit):
    def f(spec, T):
        edit(spec, T)
        return G.reference(spec, T)[0]
    return f


def _shift_tap(d):
    d["prog"][2]["dw"] += 1


def _adapter_past_ml(spec, T):
    """The adapter source's buffer holds one more tile of rows than the launch declares; the bug reads them."""
    d = copy.deepcopy(spec["desc"])
    d["a"][1]["W"] += 128
    G._fill(T.asrc(d["a"][1], 1)[..., 128:, :], torch.Generator().manual_seed(1))
    return G.reference(spec, T, desc=d)[0]


def _neighbour_range(d):
    p = d["prog"]
    p[1]["n_lo"], p[1]["n_hi"], p[2]["n_lo"], p[2]["n_hi"] = p[2]["n_lo"], p[2]["n_hi"], p[1]["n_lo"], p[1]["n_hi"]


def _last_kblock_twice(d):
    e = copy.deepcopy(d["prog"][-1])
    e["a_c0"] += 64 * (e["nchunks"] - 1)
    e["b_k0"] += 64 * (e["nchunks"] - 1)
    e["nchunks"] = 1
    d["prog"].append(e)


def _shift_bias_last_tile(spec, T):
    d = spec["desc"]
    b = T.flat(d["bias"], torch.float32)
    n0 = (d["N"] - 1) // d["block_n"] * d["block_n"]
    b[n0:d["N"]] = b[n0:d["N"]].roll(8).clone()


def _no_residual_last_tile(spec, T):
    d = spec["desc"]
    idx = T.out_index(d)[(d["M"] - 1) // 128 * 128:]
    T.flat(d["residual"], BF16)[idx] = 0


def _no_left_fill(spec, T):
    """The box of a dw = -1 tap starts in memory one pixel early instead of being zero filled: at w = 0 the
    previous image row's last pixel leaks in."""
    d = spec["desc"]
    a, W, H = d["a"][0], d["geoW"], d["geoH"]
    px = T.asrc(a, 0).double().reshape(-1, a["C"])                      # pixels in memory order
    m = torch.arange(d["M"])
    wrong = G.reference(spec, T)[0]
    pre = wrong.clone()
    if d["act"] == 0:
        for e in d["prog"]:
            if e["dw"] != -1:
                continue
            h = (m % (W * H)) // W + e["dh"]
            rows = m[(m % W == 0) & (h >= 0) & (h < H) & (m + e["dh"] * W - 1 >= 0)]
            Bm = T.bsrc(d["b"][e["b_src"]]).double()[:, e["b_k0"]:e["b_k0"] + 64 * e["nchunks"]]
            pre[rows] += d["alpha"] * px[rows + e["dh"] * W - 1][:, e["a_c0"]:e["a_c0"] + 64 * e["nchunks"]] @ Bm.t()
    return pre


def _small_adapter(corrupt):
    """The same corruption with the LoRA up-projection at 1/500 of the base weights' scale, as early in training
    (lora_B starts at zero): its whole contribution is then about half a bf16 ulp of a typical output."""
    def f(spec, T):
        T.bsrc_view(spec["desc"]["b"][1]).mul_(0.002)
        return corrupt(spec, T)
    return f


def _grouped_big():
    """grouped_spec whose adapter buffer spans one more tile of rows (poisoned) than the 128 the launch declares."""
    spec = grouped_spec(Ml=256)
    spec["desc"]["a"][1]["W"] = 128
    return spec


CORRUPTIONS = {
    "last 16 K columns of one chunk dropped": (lambda: conv3x3_spec(Cin=128), _corrupt_tensors(_drop_last16)),
    "one tap shifted by a pixel": (conv3x3_spec, _corrupt_desc(_shift_tap)),
    "no zero fill at the left image border": (conv3x3_spec, _no_left_fill),
    "adapter applied to one tile of rows past Ml": (_grouped_big, _adapter_past_ml),
    "a LoRA entry feeding its neighbour's N range": (grouped_spec, _corrupt_desc(_neighbour_range)),
    "bias shifted by 8 columns in the last N tile": (lambda: linear_spec(N=160, block_n=64), _corrupt_tensors(_shift_bias_last_tile)),
    "residual missing on the last partial M tile": (linear_spec, _corrupt_tensors(_no_residual_last_tile)),
    "last K block counted in two split-K slices": (lambda: linear_spec(K=1024, ksplit=4), _corrupt_desc(_last_kblock_twice)),
    "small adapter applied to one tile of rows past Ml": (_grouped_big, _small_adapter(_adapter_past_ml)),
    "a small LoRA entry feeding its neighbour's N range": (grouped_spec, _small_adapter(_corrupt_desc(_neighbour_range))),
}
# what the comparator of tests/test_gemm_gpu.py (a fraction of max|ref| per element, of rms(ref) on average)
# accepts of these: an adapter of realistic size in the wrong rows or columns
OLD_CLOSE_ACCEPTS = {"small adapter applied to one tile of rows past Ml", "a small LoRA entry feeding its neighbour's N range"}


def corrupted(name):
    """(spec, T, ref, S, wrong): the true reference and one corrupted the named way, on the same operands."""
    make, corrupt = CORRUPTIONS[name]
    spec = make()
    T = G.materialise(spec, CPU, seed=5)
    wrong = corrupt(spec, T)             # (a corruption that edits operands leaves the truth to be recomputed)
    if name in ("last 16 K columns of one chunk dropped", "bias shifted by 8 columns in the last N tile",
                "residual missing on the last partial M tile"):
        T = G.materialise(spec, CPU, seed=5)
    ref, S, _ = G.reference(spec, T)
    return spec, T, ref, S, wrong


@pytest.mark.parametrize("name", list(CORRUPTIONS))
def test_check_rejects_corrupted_gemm(name):
    spec, T, ref, S, wrong = corrupted(name)
    d = spec["desc"]
    assert G.check(_rounded(ref, d), ref, S, spec) <= 1.0        # the rounded truth passes
    assert (wrong != ref).any()
    with pytest.raises(AssertionError, match="outside the bound"):
        G.check(_rounded(wrong, d), ref, S, spec)


@pytest.mark.parametrize("name", list(CORRUPTIONS))
def test_which_corruptions_the_old_comparator_accepts(name):
    """The evidence that the gap was real: `_close` of test_gemm_gpu.py on the same corrupted results."""
    spec, T, ref, S, wrong = corrupted(name)
    try:
        old_suite._close(_rounded(wrong, spec["desc"]), ref.float())
        accepted = True
    except AssertionError:
        accepted = False
    assert accepted == (name in OLD_CLOSE_ACCEPTS)


@pytest.mark.parametrize("name", ["one rank column missing", "stored instead of accumulated"])
@pytest.mark.parametrize("lin", [True, False])
def test_check_rejects_corrupted_wgrad(name, lin):
    spec = wgrad_spec(lin, M=512)
    T, d = G.materialise(spec, CPU, seed=6), spec["desc"]
    ref, S, base = G.reference_wgrad(spec, T)
    out0 = T.flat(d["out"], torch.float32)[T.wgrad_index(d)].double()
    assert G.check(base, ref, S, spec, base=base) <= 1.0
    wrong = ref.clone()
    if name == "one rank column missing":
        wrong[..., 17] = out0[..., 17]
    else:
        wrong -= out0
    with pytest.raises(AssertionError, match="outside the bound"):
        G.check(wrong.float(), ref, S, spec)


def test_check_rejects_nan_and_a_worse_mean():
    spec = linear_spec()
    T = G.materialise(spec, CPU)
    ref, S, base = G.reference(spec, T)
    out = base.to(BF16)
    G.check(out, ref, S, spec, base=base)
    bad = out.clone()
    bad[7, 3] = float("nan")
    with pytest.raises(AssertionError, match="non-finite"):
        G.check(bad, ref, S, spec)
    # every element inside its bound, yet systematically off: the mean test notices
    off = ref + 0.9 * G.bound(ref, S, spec)
    with pytest.raises(AssertionError, match="twice the torch baseline"):
        G.check(off, ref, S, spec, base=base)


def test_materialise_poisons_everything_outside_the_declared_dims():
    spec = grouped_spec()
    T, d = G.materialise(spec, CPU), spec["desc"]
    out = T.flat(d["out"], BF16)
    assert out[T.out_index(d)].isnan().all()
    for b in T.bufs:
        assert (b[-G.TAIL // 2:] == G.POISON).all()
    before = G.snapshot(T)
    G.guards(spec, T, before)
    out[T.out_index(d)] = 1.0
    G.guards(spec, T, before)                      # the window may change
    out[d["M"] * d["N"]] = 1.0                     # one element past the last row
    with pytest.raises(AssertionError, match="outside the destination window"):
        G.guards(spec, T, before)


# ---------------------------------------------------------------------------------------------
# descriptor validation
# ---------------------------------------------------------------------------------------------
class Fake:
    """Stands in for materialised buffers: label i lives at a fake 256-byte aligned address."""
    ws = None

    def addr(self, ptr):
        return 0 if ptr is None else (1 << 40) + (ptr[0] << 32) + ptr[1]


@pytest.fixture(scope="module")
def lib():
    from pcm_b200 import _lib
    return _lib.lib()


def _gemm(spec, **over):
    s = G.gemm_desc(spec["desc"], Fake())
    if s.ksplit > 1 and "splitk_ws" not in over:
        s.splitk_ws = 1 << 50
    for k, v in over.items():
        setattr(s, k, v)
    return s


def _rejects(lib, rc, msg):
    assert rc != 0
    assert lib.pcm_last_error().decode() == msg


A16 = (1 << 41)
GEMM_REJECTS = [
    (dict(M=0), "pcm_gemm: M must be >= 1"),
    (dict(N=0), "pcm_gemm: N must be >= 1"),
    (dict(out=0), "pcm_gemm: out is null"),
    (dict(block_n=48), "pcm_gemm: block_n must be a multiple of 32 in [32, 256]"),
    (dict(num_prog=25), "pcm_gemm: bad source / program counts"),
    (dict(geoW=0), "pcm_gemm: geoW and geoH must be >= 1 in conv mode"),
    (dict(epiW=0), "pcm_gemm: epiW must be >= 1 in conv mode"),
    (dict(epiHW=0), "pcm_gemm: epiHW must be >= 1 in conv mode"),
    (dict(act=2), "pcm_gemm: act must be 0 or 1"),
    (dict(dep_a_src1=3), "pcm_gemm: bad dep_a_src1"),
    (dict(ksplit=4, splitk_ws=0), "pcm_gemm: ksplit > 1 needs splitk_ws"),
    (dict(ksplit=4, splitk_ws=A16 + 8), "pcm_gemm: splitk_ws is not 16-byte aligned"),
    (dict(out=A16 + 8), "pcm_gemm: out is not 16-byte aligned"),
    (dict(bias=A16 + 4), "pcm_gemm: bias is not 16-byte aligned"),
    (dict(rowvec=A16 + 2), "pcm_gemm: rowvec is not 16-byte aligned"),
    (dict(residual=A16 + 8), "pcm_gemm: residual is not 16-byte aligned"),
    (dict(osW=100), "pcm_gemm: osW is not a multiple of 8"),
    (dict(osH=804), "pcm_gemm: osH is not a multiple of 8"),
    (dict(osB=6404), "pcm_gemm: osB is not a multiple of 8"),
    (dict(rowvec=A16, rowvec_ld=100), "pcm_gemm: rowvec_ld is not a multiple of 8"),
    # elementwise epilogues (fp32 output here) only need element alignment
    (dict(out_fp32=1, out=A16 + 2), "pcm_gemm: out is not aligned to its element size"),
    (dict(out_fp32=1, bias=A16 + 2), "pcm_gemm: bias is not 4-byte aligned"),
    (dict(out_fp32=1, rowvec=A16 + 1), "pcm_gemm: rowvec is not 2-byte aligned"),
    (dict(act=1, residual=A16 + 1), "pcm_gemm: residual is not 2-byte aligned"),
    # a split-K workspace does not make the alignment irrelevant
    (dict(ksplit=4, splitk_ws=A16, act=1, out=A16 + 1), "pcm_gemm: out is not aligned to its element size"),
]


def test_gemm_rejects_what_an_unsplit_launch_would_store_misaligned(lib):
    """ksplit = 4 on a program of one K block runs unsplit, through the 16-byte epilogue."""
    spec = linear_spec(M=200, K=64, N=64, ksplit=4, residual=False)
    assert G.resolved_ksplit(spec["desc"]) == 1
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(spec))) == 0
    _rejects(lib, lib.pcm_gemm_check(ctypes.byref(_gemm(spec, out=A16 + 2))), "pcm_gemm: out is not 16-byte aligned")
    _rejects(lib, lib.pcm_gemm_check(ctypes.byref(_gemm(spec, osW=65))), "pcm_gemm: osW is not a multiple of 8")
    split = linear_spec(M=200, K=512, N=64, ksplit=4, residual=False)      # really split: elementwise finalize
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(split, out=A16 + 2, osW=65))) == 0


def test_gemm_rejects_a_misaligned_residual_prefetch(lib):
    """bf16, no activation, unsplit, 8 <= N < 32: stores are elementwise, the residual is still read 16 bytes
    at a time wherever 8 columns fit."""
    spec = linear_spec(M=200, K=64, N=24, block_n=32)
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(spec))) == 0
    _rejects(lib, lib.pcm_gemm_check(ctypes.byref(_gemm(spec, residual=A16 + 2))), "pcm_gemm: residual is not 16-byte aligned")
    _rejects(lib, lib.pcm_gemm_check(ctypes.byref(_gemm(spec, osW=25))), "pcm_gemm: osW is not a multiple of 8")
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(spec, residual=0, out=A16 + 2, osW=25))) == 0
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(linear_spec(M=200, K=64, N=4, block_n=32), residual=A16 + 2, osW=5))) == 0


@pytest.mark.parametrize("over,msg", GEMM_REJECTS, ids=[m.split(": ")[1] for _, m in GEMM_REJECTS])
def test_gemm_rejects(lib, over, msg):
    spec = conv3x3_spec()
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(spec))) == 0
    _rejects(lib, lib.pcm_gemm_check(ctypes.byref(_gemm(spec, **over))), msg)


def test_gemm_accepts_what_the_elementwise_paths_can_serve(lib):
    spec = conv3x3_spec()
    for over in (dict(out_fp32=1, out=A16 + 4, osW=100, bias=A16 + 4, rowvec=A16 + 2, rowvec_ld=101),
                 dict(act=1, out=A16 + 2, residual=A16 + 6, osW=97),
                 dict(N=24, out=A16 + 2, osW=25)):          # (conv3x3_spec has no residual)
        assert lib.pcm_gemm_check(ctypes.byref(_gemm(spec, **over))) == 0, lib.pcm_last_error()
    # N-ranged entries run unsplit: no workspace needed
    assert lib.pcm_gemm_check(ctypes.byref(_gemm(grouped_spec(), ksplit=4, splitk_ws=0))) == 0


WGRAD_REJECTS = [
    (dict(M=0), "pcm_wgrad: M must be >= 1"),
    (dict(out=0), "pcm_wgrad: out is null"),
    (dict(os_row=0), "pcm_wgrad: os_row is zero"),
    (dict(os_col=0), "pcm_wgrad: os_col is zero"),
    (dict(num_taps=10), "pcm_wgrad: bad tap count"),
    (dict(q_c0=60), "pcm_wgrad: the rank slice q[:, q_c0:] must hold a positive multiple of 8 columns"),
    (dict(out=A16 + 4), "pcm_wgrad: out is not 8-byte aligned"),
    (dict(os_row=63), "pcm_wgrad: os_row is odd with os_col == 1"),
    (dict(os_col=64, os_row=1, out=A16 + 2), "pcm_wgrad: out is not 4-byte aligned"),
    (dict(sem=A16 + 2), "pcm_wgrad: sem is not 4-byte aligned"),
]


@pytest.mark.parametrize("over,msg", WGRAD_REJECTS, ids=[m.split(": ")[1] for _, m in WGRAD_REJECTS])
def test_wgrad_rejects(lib, over, msg):
    spec = wgrad_spec(True)
    s = G._fill_struct(__import__("pcm_b200")._lib.WgradDesc(), spec["desc"], Fake())
    assert lib.pcm_wgrad_check(ctypes.byref(s)) == 0
    for k, v in over.items():
        setattr(s, k, v)
    _rejects(lib, lib.pcm_wgrad_check(ctypes.byref(s)), msg)
    s.tap_off[0] = 0


def test_wgrad_rejects_odd_tap_offset(lib):
    spec = wgrad_spec(True)
    s = G._fill_struct(__import__("pcm_b200")._lib.WgradDesc(), spec["desc"], Fake())
    s.tap_off[0] = 3
    _rejects(lib, lib.pcm_wgrad_check(ctypes.byref(s)), "pcm_wgrad: tap_off is odd with os_col == 1")


def test_the_launch_entry_points_run_the_same_checks_first():
    """Read from the source rather than by calling pcm_gemm / pcm_wgrad on fabricated addresses: each launch
    function's first statement is its validation."""
    src = open(os.path.join(os.path.dirname(_GEN), "..", "..", "pcm_b200", "csrc", "gemm_tc.cu")).read()
    for fn, check in (("launch_gemm(const pcm_gemm_desc* d, cudaStream_t stream)", "validate_gemm"),
                      ("launch_wgrad(const pcm_wgrad_desc* d, cudaStream_t stream)", "validate_wgrad")):
        body = src.split("static int " + fn + " {\n", 1)[1]
        assert body.startswith(f"  if (int rc = {check}(d)) return rc;\n"), fn


@pytest.mark.parametrize("name", list(gen.CONFIGS))
def test_every_production_launch_passes_the_validation(lib, golden, name):
    from pcm_b200 import _lib
    for spec in golden[name]:
        descs = [(spec["op"], spec["desc"])] + ([("gemm", spec["pre"])] if "pre" in spec else [])
        for op, d in descs:
            if op == "gemm":
                rc = lib.pcm_gemm_check(ctypes.byref(_gemm(dict(desc=d))))
            else:
                rc = lib.pcm_wgrad_check(ctypes.byref(G._fill_struct(_lib.WgradDesc(), d, Fake())))
            assert rc == 0, f"{lib.pcm_last_error().decode()}: {json.dumps(d, sort_keys=True)}"
