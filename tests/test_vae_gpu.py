"""The VAE on the GPU: its new kernels against float64, pcm_conv3x3_c4 / GroupNorm and the implicit GEMM at the
VAE's shapes (images 256 to 1024 pixels wide), the encoder and decoder against the oracle (oracle/vae_ref.py),
bitwise reproducibility and graph replay, the sampler's image output and the trainer's --validation_images."""
import ctypes
import gc
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_cases as GC
import test_gemm_specs_cpu as specs_cpu

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
# bf16 keeps 8 significant bits: one rounding moves a value by at most 2^-8 of its magnitude, and where an fp32 sum
# and the float64 sum fall on either side of a rounding boundary the results are one ulp, 2^-7, apart
HALF, ULP = 2.0 ** -8, 2.0 ** -7


@pytest.fixture(autouse=True)
def _exact_torch():
    """The float32 oracle runs without TF32 (it emulates bf16 products with fp32 accumulation)."""
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c
    gc.collect()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------
# new kernels against float64
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", [(3, 8), (130, 4096), (17, 16384)])
def test_softmax_rows(cuda, rows, cols):
    from pcm_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(cols)
    s = torch.randn(rows, cols + 12, device=cuda, generator=g) * 6
    s[0, :cols] += 40.0      # a large offset: the max subtraction matters
    p = torch.full((rows, cols + 4), float("nan"), device=cuda, dtype=BF)
    ops.softmax_rows(s[:, :cols], p[:, :cols])
    ref = torch.softmax(s[:, :cols].double(), -1)
    err = (p[:, :cols].double() - ref).abs()
    # bf16 rounding of the probability and fp32 exp / sum error (a few 2^-24 per term, sum of cols terms: cols
    # 2^-24 relative at most)
    assert (err <= (HALF + (cols + 8) * 2.0 ** -24) * ref + 1e-30).all(), err.max()
    assert p[:, cols:].isnan().all()


def test_transpose_bf16(cuda):
    from pcm_b200 import ops
    x = torch.randn(3, 1000, 3 * 520, device=cuda).to(BF)[:, :, 1040:]       # V columns of a q / k / v matrix
    full = torch.full((3, 520, 1000 + 8), float("nan"), device=cuda, dtype=BF)
    out = full[:, :, :1000]
    ops.transpose_bf16(x, out)
    assert torch.equal(out, x.transpose(1, 2))
    assert full[:, :, 1000:].isnan().all()


def test_latent_dist_and_sample(cuda):
    from pcm_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(0)
    B, h, w = 2, 64, 64
    hin = (torch.randn(B, h, w, 8, device=cuda, generator=g) * 3).to(BF).float()
    hin[0, 0, 0, 4:] = 100.0        # logvar clamps at 20 and -30
    hin[0, 0, 1, 4:] = -100.0
    W = (torch.randn(8, 8, device=cuda, generator=g) * 0.5).to(BF)
    W[4:, 4:] += torch.eye(4, device=cuda, dtype=BF) * 2
    b = torch.randn(8, device=cuda, generator=g) * 0.1
    mean, logvar, std = (torch.empty(B, 4, h, w, device=cuda) for _ in range(3))
    ops.latent_dist(hin, W, b, None, 1.0, mean, logvar, std, None)
    m = (hin.double().reshape(-1, 8) @ W.double().t() + b.double()).view(B, h, w, 8).permute(0, 3, 1, 2)
    # moments: one bf16 rounding of an fp32 sum of 8 products (their rounding boundary may fall either side)
    assert ((mean.double() - m[:, :4]).abs() <= ULP * m[:, :4].abs() + 1e-30).all()
    lv = m[:, 4:].clamp(-30, 20)
    assert ((logvar.double() - lv).abs() <= ULP * lv.abs() + 1e-30).all()
    assert logvar.max().item() == 20.0 and logvar.min().item() == -30.0
    sd = torch.exp(0.5 * logvar.double())
    assert ((std.double() - sd).abs() <= 4 * 2.0 ** -24 * sd).all()
    noise = torch.randn(B, 4, h, w, device=cuda, generator=g)
    out = torch.empty_like(mean)
    for scale in (1.0, 0.18215):
        ops.latent_dist(hin, W, b, noise, scale, mean, logvar, std, out)
        assert torch.equal(out, (mean + std * noise) * scale)


def test_dec_in_and_image_exit(cuda):
    from pcm_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(1)
    z = torch.randn(2, 64, 64, 4, device=cuda, generator=g) * 5
    W, b = torch.randn(4, 4, device=cuda, generator=g).to(BF), torch.randn(4, device=cuda, generator=g)
    out = torch.full((2, 64, 64, 8), float("nan"), device=cuda, dtype=BF)
    ops.vae_dec_in(z, W, b, 0.18215, out)
    x = (z / torch.tensor(0.18215, device=cuda)).to(BF).double()    # the kernel divides exactly (IEEE)
    ref = x.reshape(-1, 4) @ W.double().t() + b.double()
    assert ((out[..., :4].reshape(-1, 4).double() - ref).abs() <= ULP * ref.abs() + 1e-30).all()
    assert torch.equal(out[..., 4:], torch.zeros_like(out[..., 4:]))
    x = torch.randn(2, 96, 128, 3, device=cuda, generator=g) * 1.5
    img = torch.empty(2, 3, 96, 128, device=cuda)
    u8 = torch.empty(2, 96, 128, 3, device=cuda, dtype=torch.uint8)
    ops.image_exit(x, img, u8)
    v = (x / 2 + 0.5).clamp(0, 1)
    assert torch.equal(img, v.permute(0, 3, 1, 2))
    assert torch.equal(u8, (v * 255).round().to(torch.uint8))


# ---------------------------------------------------------------------------------------------
# existing kernels at the VAE's shapes
# ---------------------------------------------------------------------------------------------
def test_conv3x3_c4_encoder_conv_in(cuda):
    """The encoder's conv_in at 1024^2: 3 -> 128 channels (RGB with a zero fourth channel)."""
    from pcm_b200 import ops
    C, H = 128, 1024
    g = torch.Generator(device=cuda).manual_seed(C)
    x = torch.randn(1, H, H, 4, device=cuda, generator=g)
    x[..., 3] = 0
    w = (torch.randn(C, 3, 3, 4, device=cuda, generator=g) * 0.2).to(BF)
    b = torch.randn(C, device=cuda, generator=g) * 0.1
    out = torch.empty(1, H, H, C, device=cuda, dtype=BF)
    ops.conv3x3_c4(x, w, b, out)
    xr = x.to(BF).double().permute(0, 3, 1, 2)
    ref = F.conv2d(xr, w.double().permute(0, 3, 1, 2), b.double(), padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(xr.abs(), w.double().abs().permute(0, 3, 1, 2), b.double().abs(), padding=1).permute(0, 2, 3, 1)
    assert ((out.double() - ref).abs() <= HALF * ref.abs() + 40 * 2.0 ** -24 * mag).all()


@pytest.mark.parametrize("C,H,B", [(128, 1024, 1), (256, 512, 2), (512, 64, 4)])
def test_groupnorm_vae_shapes(cuda, C, H, B):
    """GroupNorm(32, eps 1e-6) + SiLU: C = 128 is 4 channels per group, an 8-wide vector spanning two groups."""
    from pcm_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C)
    x = (torch.randn(B, H * H, C, device=cuda, generator=g) * 2 + 1).to(BF)
    gamma = 1 + 0.1 * torch.randn(C, device=cuda, generator=g)
    beta = 0.1 * torch.randn(C, device=cuda, generator=g)
    out = torch.empty(B * H * H, C, device=cuda, dtype=BF)
    stats = torch.empty(B, 32, 2, device=cuda)
    ops.groupnorm_fwd(x.view(-1, C), None, gamma, beta, 1e-6, True, out, stats, B, H * H)
    y = F.group_norm(x.double().permute(0, 2, 1), 32, gamma.double(), beta.double(), 1e-6).permute(0, 2, 1)
    ref = F.silu(y).reshape(-1, C)
    assert ((out.double() - ref).abs() <= HALF * ref.abs() + 1e-4 * (1 + y.abs().reshape(-1, C))).all()


def _dec_conv_in_spec(B, h, w, Cout):
    """The decoder's conv_in as the VAE launches it: 8-channel bf16 pixels (4 of them zero), 9 taps of one
    8-wide K chunk against [Cout, 9 x 8] row-major weights."""
    from pcm_b200.unet import TAPS3

    def fn(ops):
        M = B * h * w
        ops.gemm([ops.asrc_nhwc(GC.empty((B, h, w, 8)))], [ops.bsrc(GC.empty((Cout, 72)))],
                 [(0, 0, dw, dh, 1, 0, 8 * t) for t, (dw, dh) in enumerate(TAPS3)], lin=False, M=M, N=Cout,
                 geo=(w, h), out=GC.empty((M, Cout)), bias=GC.empty((Cout,), torch.float32))
    return GC.build(fn)


@pytest.mark.parametrize("h", [64, 128])
def test_decoder_conv_in_against_float64(cuda, h):
    """Decoder conv_in (4 latent channels -> 512) on the implicit GEMM at 512^2 and 1024^2 images, against float64
    with the elementwise bound of tests/gemm_cases.py; NaN-filled surroundings stay untouched."""
    GC.run(_dec_conv_in_spec(2, h, h, 512), cuda)


def _vae_stride2_spec(B, H, W, Cin, Cout):
    from pcm_b200.vae import _S2_VAE as S2

    def fn(ops):
        x = GC.empty((B, H, W, Cin))
        planes = [x[:, p::2, q::2, :] for p in range(2) for q in range(2)]
        prog = [(S2[kh][0] * 2 + S2[kw][0], 0, S2[kw][1], S2[kh][1], Cin // 64, 0, (kh * 3 + kw) * Cin)
                for kh in range(3) for kw in range(3)]
        ops.gemm([ops.asrc_nhwc(p) for p in planes], [ops.bsrc(GC.empty((Cout, 9 * Cin)))], prog, lin=False,
                 M=B * H * W // 4, N=Cout, geo=(W // 2, H // 2), out=GC.empty((B * H * W // 4, Cout)),
                 bias=GC.empty((Cout,), torch.float32))
    return GC.build(fn)


@pytest.mark.parametrize("W", [256, 512, 1024])
def test_wide_gemm_against_float64(cuda, W):
    """3x3 pad-1 (with residual), the asymmetric stride-2 downsample and 256-row tiles at images W pixels wide,
    against float64 with the elementwise bound of tests/gemm_cases.py; NaN-filled surroundings stay untouched."""
    from pcm_b200 import _lib, ops
    GC.run(GC.conv3x3_spec(B=2, H=3, W=W, Cin=128, Cout=96, residual=True), cuda)
    GC.run(_vae_stride2_spec(2, 4, 2 * W, 64, 64), cuda)
    tall = GC.conv3x3_spec(B=1, H=67584 // W, W=W, Cin=256, Cout=128, block_n=128, ksplit=1)
    if ops.num_sms() == 132:        # H100 SXM: 528 128-row tiles take 4 waves, 264 256-row tiles 2
        assert _lib.lib().pcm_gemm_plan_rows(ctypes.byref(specs_cpu._gemm(tall))) == 256
    GC.run(tall, cuda)


def test_gemm_one_gigaelement_output(cuda):
    """The largest launch the VAE makes (MAX_LAUNCH_ELEMENTS): 16 images of 512^2 pixels, 256 output channels,
    1.07 G bf16 elements (2 GB, byte offsets past 2^31) in conv mode; rows at the start, middle and end checked
    against float64."""
    from pcm_b200 import ops
    from pcm_b200.vae import MAX_LAUNCH_ELEMENTS
    B, H, W, K, N = 16, 512, 512, 64, 256
    M = B * H * W
    assert M * N == MAX_LAUNCH_ELEMENTS
    g = torch.Generator(device=cuda).manual_seed(0)
    x = torch.randn(B, H, W, K, device=cuda, generator=g).to(BF)
    w = torch.randn(N, K, device=cuda, generator=g).to(BF)
    out = torch.empty(M, N, device=cuda, dtype=BF)
    ops.gemm([ops.asrc_nhwc(x)], [ops.bsrc(w)], [(0, 0, 0, 0, 1, 0, 0)], lin=False, M=M, N=N, geo=(W, H), out=out)
    xf = x.view(M, K)
    for r0 in (0, M // 2 - 4096, M - 8192):
        ref = xf[r0:r0 + 8192].double() @ w.double().t()
        mag = xf[r0:r0 + 8192].double().abs() @ w.double().abs().t()
        assert ((out[r0:r0 + 8192].double() - ref).abs() <= HALF * ref.abs() + 70 * 2.0 ** -24 * mag).all(), r0


# ---------------------------------------------------------------------------------------------
# the network against the oracle
# ---------------------------------------------------------------------------------------------
def _oracle(cfg_name, seed, dev):
    from oracle import vae_ref
    from pcm_b200 import vae
    cfg_o = getattr(vae_ref, cfg_name)
    P = vae_ref.init_params(cfg_o, seed)
    cfg = vae.VAEConfig(block_out_channels=cfg_o.block_out_channels, layers_per_block=cfg_o.layers_per_block)
    v = vae.AutoencoderKL(cfg, P, dev)
    emu = vae_ref.VAERef(cfg_o, {k: t.to(dev) for k, t in P.items()}, emulate_bf16=True)
    exact = vae_ref.VAERef(cfg_o, {k: t.to(dev).double() for k, t in P.items()})
    return v, emu, exact


@pytest.mark.parametrize("cfg_name,size", [("TINY", 64), ("SD15", 512)])
def test_vae_against_oracle(cuda, cfg_name, size):
    """Encoder and decoder against the bf16-emulating oracle, batch 2.  Bound: twice the emulating oracle's
    own largest distance to the float64 network (two bf16 implementations rounding at the same points, in
    different summation orders, are each that far from the exact result).  Measured own distances are printed."""
    v, emu, exact = _oracle(cfg_name, 3, cuda)
    g = torch.Generator(device=cuda).manual_seed(2)
    images = torch.rand(2, 3, size, size, device=cuda, generator=g) * 2 - 1
    with torch.no_grad():
        dist = v.encode(images).latent_dist
        me, le = emu.encode(images)
        mx, lx = exact.encode(images.double())
        own = max((me.double() - mx).abs().max().item(), (le.double() - lx).abs().max().item())
        err = max((dist.mean.double() - me).abs().max().item(), (dist.logvar.double() - le).abs().max().item())
        print(f"encode {cfg_name} {size}: |cuda - bf16 oracle| {err:.3e}, |bf16 oracle - float64| {own:.3e}")
        assert err <= 2 * own, (err, own)
        lat = torch.randn(2, 4, size // 8, size // 8, device=cuda, generator=g)
        img = v.decode(lat).sample
        re, rx = emu.decode(lat), exact.decode(lat.double())
        own = (re.double() - rx).abs().max().item()
        err = (img.double() - re).abs().max().item()
        print(f"decode {cfg_name} {size}: |cuda - bf16 oracle| {err:.3e}, |bf16 oracle - float64| {own:.3e}")
        assert err <= 2 * own, (err, own)


def test_sample_eager_graph_repeat(cuda):
    """latent_dist.sample(g) is mean + std * randn(NCHW, g) bitwise; repeated calls and a CUDA-graph replay of the
    decode are bitwise equal to eager."""
    from pcm_b200 import vae
    v = vae.AutoencoderKL.from_pretrained(None, device=cuda, config={"block_out_channels": [128, 256, 512, 512]})
    g = torch.Generator(device=cuda).manual_seed(4)
    images = torch.rand(2, 3, 256, 256, device=cuda, generator=g) * 2 - 1
    d1 = v.encode(images).latent_dist
    d2 = v.encode(images).latent_dist
    assert torch.equal(d1.mean, d2.mean) and torch.equal(d1.logvar, d2.logvar) and torch.equal(d1.std, d2.std)
    z = d1.sample(torch.Generator(device=cuda).manual_seed(7))
    n = torch.randn(d1.mean.shape, generator=torch.Generator(device=cuda).manual_seed(7), device=cuda)
    assert torch.equal(z, d1.mean + d1.std * n)
    zn = (z * v.config.scaling_factor).permute(0, 2, 3, 1).contiguous()
    eager = torch.empty(2, 3, 256, 256, device=cuda)
    u8 = torch.empty(2, 256, 256, 3, device=cuda, dtype=torch.uint8)
    v.decode_images(zn, v.config.scaling_factor, eager, u8)
    again = torch.empty_like(eager)
    v.decode_images(zn, v.config.scaling_factor, again)
    assert torch.equal(eager, again)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        v.decode_images(zn, v.config.scaling_factor, again)
    torch.cuda.current_stream().wait_stream(s)
    graph_out = torch.zeros_like(eager)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        v.decode_images(zn, v.config.scaling_factor, graph_out)
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(graph_out, eager)
    assert torch.equal(v.decode(zn.permute(0, 3, 1, 2) / 1.0).sample, v.decode(zn.permute(0, 3, 1, 2)).sample)


def test_sampler_pt_is_decode_of_latent(cuda):
    from pcm_b200 import config, weights, vae
    from pcm_b200.sampling import PCMSampler
    from pcm_b200.unet import UNetB200
    cfg = config.TINY
    net = UNetB200(cfg, weights.synthetic_state_dict(cfg, 1, lora_b_std=0.3), cuda, need_backward=False)
    v = vae.AutoencoderKL.from_pretrained(None, device=cuda, seed=2)
    smp = PCMSampler(net, vae=v)
    pe = torch.randn(2, 77, cfg.cross_attention_dim, generator=torch.Generator().manual_seed(0))
    ne = torch.zeros_like(pe)
    kw = dict(num_inference_steps=4, guidance_scale=7.5, height=128, width=128)
    lat = smp(pe, ne, generator=torch.Generator(device=cuda).manual_seed(3), **kw)
    pt = smp(pe, ne, generator=torch.Generator(device=cuda).manual_seed(3), output_type="pt", **kw)
    pt2 = smp(pe, ne, generator=torch.Generator(device=cuda).manual_seed(3), output_type="pt", **kw)
    want = torch.empty_like(pt)
    v.decode_images(lat.permute(0, 2, 3, 1).contiguous(), v.config.scaling_factor, want)
    assert pt.shape == (2, 3, 128, 128)
    assert torch.equal(pt, want) and torch.equal(pt, pt2)
    pil = smp(pe, ne, generator=torch.Generator(device=cuda).manual_seed(3), output_type="pil", **kw)
    assert len(pil) == 2 and pil[0].size == (128, 128)
    assert torch.equal(torch.from_numpy(__import__("numpy").array(pil[1])),
                       (pt[1].permute(1, 2, 0) * 255).round().to(torch.uint8).cpu())
    with pytest.raises(ValueError):
        PCMSampler(net)(pe, ne, output_type="pt", **kw)


def test_cli_validation_images(cuda, tmp_path):
    from pcm_b200 import config, ops, train_pcm_lora_sd15 as T
    vf = tmp_path / "val.pt"
    torch.save({"prompt_embeds": torch.randn(2, 77, 64, generator=torch.Generator().manual_seed(0))}, vf)
    torch.save(torch.zeros(1, 77, 64), tmp_path / "u.pt")
    ops.deterministic(True, cuda)

    def run(out, images):
        argv = ["--synthetic", "--output_dir", str(out), "--train_batch_size", "2", "--resolution", "128",
                "--multiphase", "4", "--seed", "5", "--max_train_steps", "2", "--validation_steps", "2",
                "--validation_prompt_embeds", str(vf), "--uncond_embeds", str(tmp_path / "u.pt")]
        a = T.parse_args(argv + (["--validation_images"] if images else []))
        a._cfg = config.TINY
        T.main(a)
        gc.collect()
        torch.cuda.empty_cache()

    try:
        run(tmp_path / "a", True)
        run(tmp_path / "b", False)
        from PIL import Image
        for g in (1.0, 7.5):
            d = tmp_path / "a" / "validation" / "step-2"
            pngs = sorted((d / f"cfg-{g}").glob("*.png"))
            assert len(pngs) == 8 and Image.open(pngs[0]).size == (128, 128)
            a, b = torch.load(d / f"cfg-{g}.pt"), torch.load(tmp_path / "b" / "validation" / "step-2" / f"cfg-{g}.pt")
            assert torch.equal(a["latents"], b["latents"])
        assert not (tmp_path / "b" / "validation" / "step-2" / "cfg-1.0").exists()
    finally:
        ops.deterministic(False)


def test_sdxl_1024_decode_runs(cuda):
    """A 1024^2 decode of 4 latents with the SDXL VAE config (seeded weights); prints its peak memory."""
    from pcm_b200 import vae
    v = vae.AutoencoderKL.from_pretrained(None, device=cuda, config={"scaling_factor": 0.13025}, seed=1)
    lat = torch.randn(4, 4, 128, 128, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    img = v.decode(lat / v.config.scaling_factor).sample
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"SDXL-config decode 4 x 1024^2: peak {peak / 2**30:.2f} GiB above the inputs and weights")
    assert img.shape == (4, 3, 1024, 1024) and torch.isfinite(img).all()
    assert math.isfinite(peak)
