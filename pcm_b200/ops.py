"""Thin Python wrappers over the C ABI (include/pcm_b200.h): torch tensors in, raw device pointers
across the boundary, work enqueued on torch's current CUDA stream.  No compute happens in Python.
"""
import ctypes as C
import os

import torch

from . import _lib as L

BF16 = torch.bfloat16


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def asrc_nhwc(t):
    """A-operand source from a bf16 [B, H, W, C] tensor (may be a strided view; C contiguous)."""
    assert t.dtype == BF16 and t.dim() == 4 and t.stride(3) == 1, (t.dtype, t.shape, t.stride())
    B, H, W, Cc = t.shape
    return L.ASrc(t.data_ptr(), Cc, W, H, B, t.stride(2), t.stride(1), t.stride(0))


def asrc_mat(t):
    """A-operand source from a bf16 [M, C] matrix (row stride arbitrary, C contiguous)."""
    assert t.dtype == BF16 and t.dim() == 2 and t.stride(1) == 1, (t.dtype, t.shape, t.stride())
    M, Cc = t.shape
    return L.ASrc(t.data_ptr(), Cc, M, 1, 1, t.stride(0), t.stride(0) * M, t.stride(0) * M)


def asrc_cols(a, C):
    """The same A source seen with only its first C channels (TMA zero-fills past them)."""
    return L.ASrc(a.ptr, C, a.W, a.H, a.B, a.sW, a.sH, a.sB)


def kblock(w):
    """[N, K] row-major -> K-blocked [K/64, N, 64] (see pcm_bsrc.kblocked): the frozen weights are
    stored this way so that the N x 64 operand tile of a K block is contiguous in HBM."""
    N, K = w.shape
    assert K % 64 == 0
    return w.reshape(N, K // 64, 64).permute(1, 0, 2).contiguous()


def bsrc(w):
    """B-operand source from bf16 weights: [N, K] row-major (K contiguous) or K-blocked [K/64, N, 64]."""
    if w.dim() == 3:
        assert w.dtype == BF16 and w.is_contiguous() and w.shape[2] == 64, (w.dtype, w.shape, w.stride())
        return L.BSrc(w.data_ptr(), w.shape[0] * 64, w.shape[1], 64, 1)
    assert w.dtype == BF16 and w.dim() == 2 and w.stride(1) == 1, (w.dtype, w.shape, w.stride())
    return L.BSrc(w.data_ptr(), w.shape[1], w.shape[0], w.stride(0), 0)


_NUM_SMS = None
# kernel-launch accounting (bench.py `gpu_launches`) and optional per-launch GEMM profiling
LAUNCHES = {"count": 0}
PROFILE = None  # list of (start_event, end_event, flops) when enabled
PROFILE_EXTERNAL = False  # True: events become event-record NODES when captured in a CUDA graph
DRY_RUN = None  # list: record (kind, info) instead of launching (shape analysis without a GPU)
_KERNELS_PER_CALL = {"pcm_groupnorm_fwd": 2, "pcm_groupnorm_fwd_part": 2, "pcm_groupnorm_bwd": 2, "pcm_attn_bwd": 3, "pcm_adamw_clip": 2}



def num_sms():
    global _NUM_SMS
    if _NUM_SMS is None:
        _NUM_SMS = 132 if DRY_RUN is not None else L.lib().pcm_num_sms()
    return _NUM_SMS


def pick_block_n(M, N):
    """N tile (multiple of 32, <= 256) minimising waves x tile width on the persistent grid."""
    tiles_m = (M + 127) // 128
    sms = num_sms()
    best, best_cost = None, None
    for bn in (256, 224, 192, 160, 128, 96, 64, 32):
        if bn > 32 and bn - 32 >= N:
            continue
        tiles = tiles_m * ((N + bn - 1) // bn)
        waves = (tiles + sms - 1) // sms
        cost = waves * (bn + 24)  # +24: per-tile fixed cost (epilogue drain, pipeline fill)
        if best_cost is None or cost < best_cost:
            best, best_cost = bn, cost
    return best


def pick_tiling(M, N, nkb):
    """(block_n, ksplit): small-M long-K GEMMs (the 8x8 / 16x16 UNet levels, LoRA-A convs) leave most
    SMs idle with one CTA per output tile, so their K loop is split over several CTAs."""
    sms = num_sms()
    tiles_m = (M + 127) // 128
    if nkb >= 32:
        bn = min(256, ((N + 31) // 32) * 32)          # widest tile: best operand reuse
        tiles = tiles_m * ((N + bn - 1) // bn)
        if tiles * 2 <= sms:
            ks = min(nkb // 8, sms // tiles)
            if ks >= 2:
                return bn, ks
    return pick_block_n(M, N), 1


def chunk_widths(a_srcs, b_srcs, e):
    """K columns each 64-wide chunk of K-program entry e multiplies: those both operands have,
    min(64, a.C - (a_c0 + 64c), b.K - (b_k0 + 64c)) (a LoRA rank r % 64 != 0 ends the last chunk early;
    the kernel rounds the width up to 16, multiplying TMA-filled zeros)."""
    kend = min(a_srcs[e[0]].C - e[5], b_srcs[e[1]].K - e[6])
    return [max(0, min(64, kend - 64 * c)) for c in range(e[4])]


def gemm_flops(a_srcs, prog, M, N, lin, geo, b_srcs=None):
    """ALGORITHMIC flops of one launch: an N-ranged K entry only counts its own output columns, an A
    source with fewer rows than the output (the LoRA T of the leading samples) only its own rows, and a
    chunk only the K columns both operands have (with b_srcs)."""
    fl = 0.0
    for e in prog:
        a = a_srcs[e[0]]
        rows = min(M, a.W if lin else a.B * geo[0] * geo[1])
        cols = min(N, e[8] - e[7]) if (len(e) > 7 and e[8]) else N
        k = 64 * e[4] if b_srcs is None else sum(chunk_widths(a_srcs, b_srcs, e))
        fl += 2.0 * rows * cols * k
    return fl


def gemm(a_srcs, b_srcs, prog, *, lin, M, N, out, geo=(1, 1), bias=None, rowvec=None,
         residual=None, out_strides=None, epi=None, alpha=1.0, act=0, round_bf16=False,
         block_n=None, ksplit=None, dep_a_src=None, splitk_ws=None):
    """Launch the wgmma implicit GEMM.  prog: list of (a_src, b_src, dw, dh, nchunks, a_c0, b_k0
    [, n_lo, n_hi]); an entry with n_hi > 0 only feeds output columns [n_lo, n_hi).

    dep_a_src: index of the A source that the launch issued IMMEDIATELY before this one produced (the
    layer's LoRA down-projection); the kernel then only waits for that launch right before reading it.

    out: bf16 or fp32 tensor; rows are addressed as b*osB + h*osH + w*osW with (osW, osH, osB) =
    out_strides (default: dense [M, ld] with ld = out.stride(-2))."""
    d = L.GemmDesc()
    for i, a in enumerate(a_srcs):
        d.a[i] = a
    for i, b in enumerate(b_srcs):
        d.b[i] = b
    for i, e in enumerate(prog):
        d.prog[i] = L.KEntry(*e[:7], *(e[7:9] if len(e) > 7 else (0, 0)))
    d.num_a, d.num_b, d.num_prog = len(a_srcs), len(b_srcs), len(prog)
    d.lin, d.M, d.N = int(lin), M, N
    d.geoW, d.geoH = geo
    nkb = sum(e[4] for e in prog)
    if any(len(e) > 7 and e[8] for e in prog):
        ksplit = 1
        assert block_n is not None
    if block_n is None and ksplit is None:
        block_n, ksplit = pick_tiling(M, N, nkb)
    d.block_n = block_n or pick_block_n(M, N)
    d.ksplit = ksplit or 1
    ws = None
    if d.ksplit > 1:
        # one fp32 slice per K split (plain stores, added in split order by the finalize kernel)
        ws = splitk_ws
        if ws is None and DRY_RUN is None:
            ws = torch.empty(d.ksplit, M, N, device=out.device, dtype=torch.float32)
        d.splitk_ws = ws.data_ptr() if ws is not None else 0
    d.out = out.data_ptr()
    d.out_fp32 = int(out.dtype == torch.float32)
    assert out.dtype in (torch.float32, BF16)
    d.round_bf16 = int(round_bf16)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() >= N
        d.bias = bias.data_ptr()
    if rowvec is not None:
        assert rowvec.dtype == BF16 and rowvec.stride(-1) == 1
        d.rowvec = rowvec.data_ptr()
        d.rowvec_ld = rowvec.stride(0)
    if residual is not None:
        assert residual.dtype == BF16
        d.residual = residual.data_ptr()
    if out_strides is None:
        ld = out.stride(-2)
        if lin:
            out_strides, epi = (ld, 0, 0), (1 << 30, 1 << 30)
        else:
            W, H = geo
            out_strides, epi = (ld, ld * W, ld * W * H), (W, W * H)
    d.osW, d.osH, d.osB = out_strides
    d.epiW, d.epiHW = epi
    d.alpha = alpha
    d.act = act
    d.dep_a_src1 = 0 if dep_a_src is None else dep_a_src + 1
    LAUNCHES["count"] += 1
    if DRY_RUN is not None:
        DRY_RUN.append(("gemm", dict(M=M, N=N, K=64 * sum(e[4] for e in prog), bn=d.block_n, lin=int(lin),
                                     nprog=len(prog), res=residual is not None, ksplit=d.ksplit,
                                     prog=[tuple(e) for e in prog], num_a=len(a_srcs), num_b=len(b_srcs),
                                     a_C=[a.C for a in a_srcs], b_K=[b.K for b in b_srcs],
                                     b_N=[b.N for b in b_srcs], dep=dep_a_src,
                                     flop=gemm_flops(a_srcs, prog, M, N, lin, geo, b_srcs))))
        return out
    if PROFILE is not None:
        e0 = torch.cuda.Event(enable_timing=True, external=PROFILE_EXTERNAL)
        e1 = torch.cuda.Event(enable_timing=True, external=PROFILE_EXTERNAL)
        e0.record()
        L.check(L.lib().pcm_gemm(C.byref(d), _stream()), "pcm_gemm")
        e1.record()
        PROFILE.append((e0, e1, gemm_flops(a_srcs, prog, M, N, lin, geo, b_srcs)))
        return out
    L.check(L.lib().pcm_gemm(C.byref(d), _stream()), "pcm_gemm")
    return out


TAPS3 = [(kw - 1, kh - 1) for kh in range(3) for kw in range(3)]  # (dw, dh), tap = kh*3 + kw


# int32 semaphores for reproducible LoRA weight gradients (pcm_wgrad_desc.sem): the token splits of
# a wgrad tile then accumulate in split order
WGRAD_SEM = None
_DET = os.environ.get("PCM_DETERMINISTIC", "0") == "1"


def deterministic(on, device=None):
    """Bit-reproducible mode.  GroupNorm statistics, split-K, the gradient norm and the loss
    reduction are always order independent; the LoRA weight gradients (token-split fp32 `red`)
    additionally need this switch (or PCM_DETERMINISTIC=1), which serialises the splits of a tile."""
    global WGRAD_SEM, _DET
    _DET = bool(on)
    WGRAD_SEM = torch.zeros(4096, device=device or "cuda", dtype=torch.int32) if on else None


def wgrad(p_src, q_src, out, *, lin, M, geo=(1, 1), taps=((0, 0),), tap_off=(0,), os_row, os_col,
          alpha=1.0, q_c0=0, ksplit=0):
    """out[tap_off[t] + ch*os_row + r*os_col] += alpha * sum_m P[m(+tap t), ch] * Q[m, q_c0 + r]."""
    assert out.dtype == torch.float32
    d = L.WgradDesc()
    d.p, d.q = p_src, q_src
    d.q_c0, d.lin, d.M = q_c0, int(lin), M
    d.geoW, d.geoH = geo
    d.num_taps = len(taps)
    for i, (dw, dh) in enumerate(taps):
        d.dw[i], d.dh[i] = dw, dh
        d.tap_off[i] = tap_off[i]
    d.out = out.data_ptr()
    d.os_row, d.os_col = os_row, os_col
    d.ksplit = ksplit
    d.alpha = alpha
    if _DET and DRY_RUN is None:
        if WGRAD_SEM is None:
            deterministic(True)
        assert ((p_src.C + 127) // 128) * len(taps) <= WGRAD_SEM.numel()
        d.sem = WGRAD_SEM.data_ptr()
    LAUNCHES["count"] += 1
    if DRY_RUN is not None:
        DRY_RUN.append(("wgrad", dict(M=M, Cp=p_src.C, taps=len(taps))))
        return out
    L.check(L.lib().pcm_wgrad(C.byref(d), _stream()), "pcm_wgrad")
    return out


# ---------------------------------------------------------------------------------------------
# normalisation / attention / glue / PCM math / optimiser wrappers
# ---------------------------------------------------------------------------------------------
def _p(t):
    return t.data_ptr() if t is not None else None


def _call(name, *args):
    LAUNCHES["count"] += _KERNELS_PER_CALL.get(name, 1)
    if DRY_RUN is not None:
        DRY_RUN.append((name, None))
        return
    L.check(getattr(L.lib(), name)(*args, torch.cuda.current_stream().cuda_stream), name)


_GN_WS = {}


def gn_workspace(device, B, HW, C, G):
    """Per-device GroupNorm scratch (block counters + per-block partial statistics), zero-initialised
    once and grown on demand; the kernels leave the counters at zero."""
    if DRY_RUN is not None:
        return None, 0
    need = L.lib().pcm_groupnorm_ws_bytes(B, HW, C, G)
    if need < 0:
        raise L.PcmError(L.lib().pcm_last_error().decode())
    key = torch.device(device)
    ws = _GN_WS.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(max(need, 8 << 20), device=device, dtype=torch.uint8)
        _GN_WS[key] = ws
    return ws, ws.numel()


def groupnorm_fwd(x1, x2, gamma, beta, eps, silu, out, stats, B, HW, G=32):
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    ws, nws = gn_workspace(x1.device, B, HW, C1 + C2, G)
    _call("pcm_groupnorm_fwd", _p(x1), _p(x2), C1, C2, B, HW, G, _p(gamma), _p(beta), eps, int(silu),
          _p(out), _p(stats), _p(ws), nws)
    return out


def groupnorm_fwd_part(x1, x2, gamma, beta, eps, silu, out, stats, B, part_B, HW, G=32):
    """groupnorm_fwd over B images, with the per-image block partition of a launch over part_B >= B
    images: bitwise equal to rows 0..B-1 of that launch (a block rebuilt for the backward from the
    leading samples of a merged batch)."""
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    ws, nws = gn_workspace(x1.device, B, HW, C1 + C2, G)
    _call("pcm_groupnorm_fwd_part", _p(x1), _p(x2), C1, C2, B, part_B, HW, G, _p(gamma), _p(beta), eps,
          int(silu), _p(out), _p(stats), _p(ws), nws)
    return out


def groupnorm_bwd(dy, x1, x2, gamma, beta, eps, silu, stats, red, add, dx1, dx2, B, HW, G=32, colsum=None):
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    ws, nws = gn_workspace(x1.device, B, HW, C1 + C2, G)
    _call("pcm_groupnorm_bwd", _p(dy), _p(x1), _p(x2), C1, C2, B, HW, G, _p(gamma), _p(beta), eps,
          int(silu), _p(stats), _p(red), _p(add), _p(dx1), _p(dx2), _p(colsum), _p(ws), nws)


def cast_f32_bf16(x, out):
    _call("pcm_cast_f32_bf16", _p(x), x.numel(), _p(out))
    return out


def layernorm_fwd(x, gamma, beta, out, stats, eps=1e-5):
    M, Cc = x.shape
    _call("pcm_layernorm_fwd", _p(x), M, Cc, _p(gamma), _p(beta), eps, _p(out), _p(stats))
    return out


def layernorm_bwd(dy, x, gamma, stats, add, dx):
    M, Cc = x.shape
    _call("pcm_layernorm_bwd", _p(dy), _p(x), M, Cc, _p(gamma), _p(stats), _p(add), _p(dx))
    return dx


def attn_fwd(q, k, v, out, lse, B, H, Sq, Skv, D, scale):
    """q/out: [B*Sq, >=H*D] views, k/v: [B*Skv, >=H*D] views (row stride = .stride(0))."""
    _call("pcm_attn_fwd", _p(q), _p(k), _p(v), _p(out), _p(lse), B, H, Sq, Skv, D, q.stride(0),
          k.stride(0), v.stride(0), out.stride(0), scale)
    return out


def attn_bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, B, H, Sq, Skv, D, scale):
    assert o.stride(0) == dout.stride(0) and dq.stride(0) == q.stride(0)
    assert dk.stride(0) == k.stride(0) and dv.stride(0) == v.stride(0)
    _call("pcm_attn_bwd", _p(q), _p(k), _p(v), _p(o), _p(dout), _p(lse), _p(delta), _p(dq), _p(dk),
          _p(dv), B, H, Sq, Skv, D, q.stride(0), k.stride(0), v.stride(0), o.stride(0), scale)


def geglu_fwd(u, out):
    M, F2 = u.shape
    _call("pcm_geglu_fwd", _p(u), M, F2 // 2, _p(out))
    return out


def geglu_bwd(dgg, u, du):
    M, F2 = u.shape
    _call("pcm_geglu_bwd", _p(dgg), _p(u), M, F2 // 2, _p(du))
    return du


def upsample2x_fwd(x, out):
    B, H, W, Cc = x.shape
    _call("pcm_upsample2x_fwd", _p(x), B, H, W, Cc, _p(out))
    return out


def upsample2x_bwd(dout, din):
    B, H, W, Cc = din.shape
    _call("pcm_upsample2x_bwd", _p(dout), B, H, W, Cc, _p(din))
    return din


def conv3x3_c4(x, w, bias, out, sgn=1, round_in=True):
    B, H, W, four = x.shape
    assert four == 4 and x.dtype == torch.float32
    _call("pcm_conv3x3_c4", _p(x), B, H, W, out.shape[-1], _p(w), _p(bias), sgn, int(round_in), _p(out))
    return out


def softmax_rows(s, p):
    """p = bf16(softmax(s, -1)), fp32 max and sum: s fp32 [rows, cols], p bf16 [rows, cols] (row strides free)."""
    assert s.dtype == torch.float32 and p.dtype == BF16 and s.shape == p.shape and s.stride(1) == p.stride(1) == 1
    _call("pcm_softmax_rows", _p(s), s.shape[0], s.shape[1], s.stride(0), _p(p), p.stride(0))
    return p


def transpose_bf16(x, out):
    """out[b] = x[b]^T for bf16 [batch, rows, cols] -> [batch, cols, rows] (row and batch strides free)."""
    assert x.dtype == out.dtype == BF16 and x.stride(2) == out.stride(2) == 1
    batch, rows, cols = x.shape
    assert tuple(out.shape) == (batch, cols, rows)
    _call("pcm_transpose_bf16", _p(x), rows, cols, x.stride(1), x.stride(0), batch, _p(out), out.stride(1),
          out.stride(0))
    return out


def latent_dist(h, w, bias, noise, scale, mean, logvar, std, sample):
    """quant_conv + DiagonalGaussianDistribution: h fp32 [B, hh, ww, 8]; mean / logvar / std (/ sample with
    noise) fp32 NCHW [B, 4, hh, ww]."""
    B, hh, ww, eight = h.shape
    assert eight == 8 and h.dtype == torch.float32 and h.is_contiguous() and mean.is_contiguous()
    assert noise is None or (noise.is_contiguous() and noise.shape == mean.shape)
    _call("pcm_latent_dist", _p(h), B, hh * ww, _p(w), _p(bias), _p(noise), scale, _p(mean), _p(logvar), _p(std),
          _p(sample))


def vae_dec_in(z, w, bias, div, out):
    """post_quant_conv on z / div: z fp32 NHWC [B, h, w, 4] -> out bf16 NHWC [B, h, w, 8], channels 4..7 zero."""
    assert z.dtype == torch.float32 and out.dtype == BF16 and z.is_contiguous() and out.is_contiguous()
    assert z.shape[-1] == 4 and tuple(out.shape) == tuple(z.shape[:-1]) + (8,)
    _call("pcm_vae_dec_in", _p(z), z.numel() // 4, _p(w), _p(bias), div, _p(out))
    return out


def image_exit(x, out, u8=None):
    """(x / 2 + 0.5).clamp(0, 1): x fp32 NHWC [B, H, W, C] -> out fp32 NCHW (or None), u8 uint8 NHWC (or None)."""
    B, H, W, Cc = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    assert out is None or (out.is_contiguous() and tuple(out.shape) == (B, Cc, H, W))
    assert u8 is None or (u8.dtype == torch.uint8 and u8.is_contiguous() and u8.shape == x.shape)
    _call("pcm_image_exit", _p(x), B, H * W, Cc, _p(out), _p(u8))
    return out


def timestep_embed(t, out):
    _call("pcm_timestep_embed", _p(t), out.shape[0], out.shape[1], _p(out))
    return out


def colsum(x, out, B, HW):
    _call("pcm_colsum", _p(x), B, HW, x.shape[-1], _p(out))
    return out


def add_bf16(a, b, out):
    _call("pcm_add_bf16", _p(a), _p(b), a.numel(), _p(out))
    return out


def lora_fuse(master, table, work, scale):
    """W + scale * B A into the destinations of `table` (UNetB200.fused_inference_net), from the fp32
    masters `master`."""
    assert master.dtype == torch.float32 and table.dtype == torch.int64 and table.shape[1] == 8
    _call("pcm_lora_fuse", _p(master), _p(table), table.shape[0], work, scale)


def sample_step(eps, x, out, out2, guidance, sa, ss, sap, ssp, pred_type):
    """One eta = 0 DDIM step on fp32 latents x [B, ...].  guidance: None, or a float64 device scalar g
    (eps is then the [uncond; cond] batch [2B, ...], mixed eps_u + g (eps_c - eps_u))."""
    B = x.shape[0]
    per = x.numel() // B
    cfg = guidance is not None
    assert eps.shape[0] == (2 * B if cfg else B) and eps.dtype == x.dtype == torch.float32
    assert not cfg or guidance.dtype == torch.float64
    _call("pcm_sample_step", _p(eps), _p(x), _p(out), _p(out2), per, B, int(cfg), _p(guidance), sa, ss, sap,
          ssp, pred_type)
    return out
