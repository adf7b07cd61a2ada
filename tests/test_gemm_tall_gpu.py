"""The implicit GEMM's 256-row tiles: two 128-row A slabs per stage against one weight tile.

* CPU: which launches pcm_gemm_plan_rows sends to 256-row tiles, on hand-built descriptors and on every
  recorded launch of the SD1.5 / SDXL steps (never a split-K launch, a block_n other than 128 / 160, fewer
  than 32 K blocks per tile, or an M-ranged entry that ends inside a 256-row tile).
* GPU: launches that take 256-row tiles agree bit for bit with the same rows computed by a launch that takes
  128-row tiles (the rows of a 2048-row slice of a Linear, one image of a 24-image convolution), and pass the
  float64 check with NaN-guarded buffers (gemm_cases.run)."""
import copy
import ctypes

import pytest
import torch

import gemm_cases
import gemm_spec as G
import test_gemm_specs_cpu as specs_cpu
from gemm_cases import concat_lora_spec, conv3x3_spec, dgrad2_spec, linear_spec, stride2_spec

SMS = 132   # the H100 SXM count the rule is pinned at (num_sms() without a device, too)
MIN_KB = 32
K = 64 * MIN_KB


@pytest.fixture(scope="module")
def lib():
    from pcm_b200 import _lib
    return _lib.lib()


def plan_rows(lib, spec, **over):
    return lib.pcm_gemm_plan_rows(ctypes.byref(specs_cpu._gemm(spec, **over)))


def rule(M, N, bn):
    """The wave rule of gemm_plan_rows, written out."""
    tn = -(-N // bn)
    w128, w256 = -(-(-(-M // 128) * tn) // SMS), -(-(-(-M // 256) * tn) // SMS)
    return 256 if 2 * w256 <= w128 else 128


# ---------------------------------------------------------------------------------------------
# CPU: the rule
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [2048, 16896, 33792, 33792 + 128, 65344, 65408, 65472, 98304])
@pytest.mark.parametrize("bn", [128, 160])
def test_wave_rule(lib, M, bn):
    assert plan_rows(lib, linear_spec(M, K, 320, block_n=bn)) == rule(M, 320, bn)


def test_rule_cases(lib):
    assert plan_rows(lib, linear_spec(98304, K, 320, block_n=160)) == 256
    assert plan_rows(lib, linear_spec(98304, K - 64, 320, block_n=160)) == 128      # too short a K loop
    assert plan_rows(lib, linear_spec(98304, K - 64, 320, block_n=160, rank=64)) == 256   # + the LoRA block
    assert plan_rows(lib, linear_spec(2048, K, 320, block_n=160)) == 128              # one wave either way
    for bn in (32, 64, 96, 192, 224, 256):                                            # no 256-row kernel
        assert plan_rows(lib, linear_spec(98304, K, 320, block_n=bn)) == 128, bn
    # a K split that really runs keeps 128-row tiles
    assert plan_rows(lib, linear_spec(98304, K, 320, block_n=160, ksplit=4), splitk_ws=1 << 50) == 128
    # M-ranged LoRA entries: the A source must end on a 256-row tile boundary, and its K blocks do not count
    assert plan_rows(lib, linear_spec(98304, K, 320, block_n=160, rank=64, Ml=49152)) == 256
    assert plan_rows(lib, linear_spec(98304, K - 64, 320, block_n=160, rank=64, Ml=49152)) == 128
    assert plan_rows(lib, linear_spec(98304, K, 320, block_n=160, rank=64, Ml=49152 + 128)) == 128
    # an A source with fewer rows that is not a whole number of 128-row tiles is not M-ranged at all
    assert plan_rows(lib, linear_spec(98304, K, 320, block_n=160, rank=64, Ml=49152 + 64)) == 256
    # N-ranged entries feed some tiles only: their K blocks do not count
    spec = linear_spec(98304, K - 64, 320, block_n=160, rank=64, ranged=(0, 160))
    assert plan_rows(lib, spec) == 128


@pytest.mark.parametrize("name", list(specs_cpu.gen.CONFIGS))
def test_recorded_launches(lib, name):
    """Every recorded launch: 256 rows exactly where the rule allows them."""
    tall = 0
    for spec in G.trace.load(specs_cpu.gen.FIXTURE)[name]:
        if spec["op"] != "gemm":
            continue
        for d in [spec["desc"]] + ([spec["pre"]] if "pre" in spec else []):
            rows = plan_rows(lib, dict(desc=d))
            m_hi = [G._m_hi(d, e) for e in d["prog"]]
            nkb = sum(e["nchunks"] for e, m in zip(d["prog"], m_hi) if not e["n_hi"] and not m)
            allowed = (d["block_n"] in (128, 160) and G.resolved_ksplit(d) == 1 and all(m % 256 == 0 for m in m_hi)
                       and nkb >= MIN_KB)
            assert rows == (rule(d["M"], d["N"], d["block_n"]) if allowed else 128), d
            tall += rows == 256
    assert tall >= 30, tall    # the BN = 160 level-0/1 3x3 convolutions, long Linears and their dgrads


# ---------------------------------------------------------------------------------------------
# GPU: bitwise against 128-row tiles, float64 check
# ---------------------------------------------------------------------------------------------
def rows_of(d, r0, m):
    """Rows r0 .. r0 + m - 1 of launch d as a launch of their own: A sources, output, residual and row
    vector advanced to row r0 (an image boundary in conv mode)."""
    d = copy.deepcopy(d)
    per = 1 if d["lin"] else d["geoW"] * d["geoH"]
    assert r0 % per == 0 and (r0 % d["epiHW"] == 0 or d["epiHW"] > d["M"])
    for a in d["a"]:
        if d["lin"]:
            a["ptr"][1] += 2 * r0 * a["sW"]
            a["W"] -= r0
        else:
            a["ptr"][1] += 2 * (r0 // per) * a["sB"]
            a["B"] -= r0 // per
        assert (a["W"] if d["lin"] else a["B"] * per) >= m
    off, b = G._row_offsets(r0 + 1, d["epiW"], d["epiHW"], d["osW"], d["osH"], d["osB"])
    d["out"][1] += (4 if d["out_fp32"] else 2) * int(off[r0])
    if d["residual"]:
        d["residual"][1] += 2 * int(off[r0])
    if d["rowvec"]:
        d["rowvec"][1] += 2 * int(b[r0]) * d["rowvec_ld"]
    d["M"] = m
    return d


def tall_vs_short(spec, device, slices):
    """Run the spec (256-row tiles) with the float64 check, then each (r0, m) row slice as a launch of its own
    (128-row tiles) into a NaN-filled window: the slice's rows must be bit-identical."""
    from pcm_b200 import _lib
    lib = _lib.lib()
    assert plan_rows(lib, spec) == 256
    T = G.materialise(spec, device)
    out = gemm_cases.run_and_check(spec, T, G.snapshot(T)).clone()
    for r0, m in slices:
        sub = rows_of(spec["desc"], r0, m)
        s = G.gemm_desc(sub, T)
        assert lib.pcm_gemm_plan_rows(ctypes.byref(s)) == 128
        flat, idx = G.window(dict(op="gemm", desc=sub), T)
        flat[idx] = float("nan")
        _lib.check(lib.pcm_gemm(ctypes.byref(s), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pcm_gemm")
        torch.cuda.synchronize()
        got = flat[idx]
        want = out[r0:r0 + m]
        assert torch.equal(got.view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32),
                           want.view(torch.int16 if want.dtype == torch.bfloat16 else torch.int32)), (r0, m)


def lin_slices(M):
    return [(0, 2048), (M - 2048, 2048)]


def conv_slices(B, H, W):
    return [(0, H * W), ((B - 1) * H * W, H * W)]


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [0, 64, 128, 192], ids=lambda t: f"M%256={t}")
def test_linear_residual_bias(cuda, tail):
    M = 65280 + tail if tail else 98304
    spec = linear_spec(M, K, 320, block_n=160, residual=True)
    tall_vs_short(spec, cuda, lin_slices(M))


@pytest.mark.gpu
@pytest.mark.parametrize("out", ["bf16", "fp32", "round"])
def test_linear_rowvec_silu(cuda, out):
    M = 65536
    spec = linear_spec(M, K, 320, block_n=160, rowvec=True, act=1, out=out, alpha=0.5)
    tall_vs_short(spec, cuda, lin_slices(M))


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 160])
@pytest.mark.parametrize("rank", [64, 32, 96], ids=lambda r: f"r{r}")
def test_linear_lora(cuda, bn, rank):
    """A fused LoRA K block on every row (r = 32, 96: NARROW kernels)."""
    M = 65536
    tall_vs_short(linear_spec(M, K, 640 if bn == 128 else 320, block_n=bn, rank=rank), cuda, lin_slices(M))


@pytest.mark.gpu
@pytest.mark.parametrize("dep", [False, True], ids=["plain", "dep_a_src1"])
def test_linear_m_ranged_lora(cuda, dep):
    """The LoRA T of the leading 32768 rows only (M-ranged entry), produced by the launch before (dep_a_src1:
    tiles visited last-to-first, late wait on T)."""
    M, Ml = 65536, 32768
    spec = linear_spec(M, K, 320, block_n=160, rank=32, Ml=Ml, dep=dep)
    assert [G._m_hi(spec["desc"], e) for e in spec["desc"]["prog"]] == [0, Ml]
    tall_vs_short(spec, cuda, [(0, 2048), (Ml - 2048, 2048)])


@pytest.mark.gpu
def test_conv3x3(cuda):
    B, H, W = 24, 64, 64
    tall_vs_short(conv3x3_spec(B, H, W, 256, 320, rowvec=True, residual=True), cuda, conv_slices(B, H, W))


@pytest.mark.gpu
def test_conv3x3_ragged_batch(cuda):
    """8 x 8 images: a 256-row tile spans four images, and the last tile's second slab lies past the batch."""
    B, H, W = 1046, 8, 8                       # M = 66944 = 261 * 256 + 128
    spec = conv3x3_spec(B, H, W, 256, 320, rowvec=True, residual=True)
    assert spec["desc"]["M"] % 256 == 128
    tall_vs_short(spec, cuda, conv_slices(B, H, W))


@pytest.mark.gpu
def test_skip_concat_lora(cuda):
    """Two K segments (skip concat) plus a narrow LoRA K block, fp32 output."""
    B, H, W = 24, 64, 64
    spec = concat_lora_spec(B, H, W, C1=256, C2=128, Cout=320, r=24)
    tall_vs_short(spec, cuda, conv_slices(B, H, W))


@pytest.mark.gpu
def test_stride2_planes(cuda):
    B, H, W = 24, 128, 128
    tall_vs_short(stride2_spec(B, H, W, 256, 320), cuda, conv_slices(B, H // 2, W // 2))


@pytest.mark.gpu
def test_dgrad2_strided_plane(cuda):
    """Input gradient of the stride-2 convolution stored into one parity plane, with a narrow LoRA block."""
    B, H, W = 24, 128, 128
    spec = dgrad2_spec(1, 1, B, H, W, Cin=320, Cout=512, rank=24)
    tall_vs_short(spec, cuda, conv_slices(B, H // 2, W // 2))
