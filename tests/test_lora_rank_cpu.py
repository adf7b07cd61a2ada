"""LoRA adapters of any supported rank (8 <= r <= 256, r % 8 == 0) on the HOST side, on CPU.

The kernels' rank rules, restated here as an interpreter of the launch descriptors:
  * a pcm_gemm K chunk multiplies only the K columns both operands have,
    min(64, a.C - (a_c0 + 64c), b.K - (b_k0 + 64c)) (TMA zero-fills the operand that ends first);
  * a pcm_wgrad launch covers the rank slice q[:, q_c0:q_c0 + w], w = min(64, q.C - q_c0), and stores
    only those w columns;
  * pcm_lora_refresh works in min(r, 64) x 64 tiles, ceil(r / 64) rank tiles per 64 columns.
The UNet's launch plans run through that interpreter (and the torch semantics of every other kernel,
tests/ops_interp.py) and are compared with the oracle network at several ranks."""
import dataclasses
import math

import pytest
import torch

import ops_interp
from gemm_interp import BF16, a_nhwc, b_matrix, mat, refresh_operands, shifted_rows

RECORD = None   # list: (kind, info) of every interpreted launch while a test collects them


def interp_gemm_any(a_srcs, b_srcs, prog, *, lin, M, N, out, geo=(1, 1), bias=None, residual=None, act=0,
                    rowvec=None, alpha=1.0, round_bf16=False, block_n=None, **kw):
    from pcm_b200 import ops
    Wo, Ho = geo
    Bo = M // (Wo * Ho)
    acc = torch.zeros(M, N, dtype=torch.float32)
    for e in prog:
        a, b = a_srcs[e[0]], b_srcs[e[1]]
        assert e[6] % (64 if b.kblocked else 8) == 0, e
        widths = ops.chunk_widths(a_srcs, b_srcs, e)
        assert all(w == 64 for w in widths[:-1]) and widths[-1] > 0, (e, widths)
        if RECORD is not None:
            RECORD.append(("gemm", dict(entry=tuple(e), widths=widths, a_C=a.C, b_K=b.K, block_n=block_n, N=N)))
        kk = sum(widths)
        lo, hi = (e[7], e[8]) if (len(e) > 7 and e[8]) else (0, N)
        if len(e) > 7 and e[8]:
            assert block_n is not None and lo % block_n == 0 and (hi % block_n == 0 or hi >= N), (e, block_n)
        Bm = b_matrix(b)[lo:hi, e[6]:e[6] + kk].float()
        if lin:
            rows = min(M, a.W)
            A = mat(a.ptr, rows, a.C, a.sW)[:, e[5]:e[5] + kk].float()
            acc[:rows, lo:hi] += A @ Bm.t()
        else:
            A = shifted_rows(a, e[2], e[3], Wo, Ho, Bo)[:, e[5]:e[5] + kk]
            acc[:, lo:hi] += A @ Bm.t()
    acc = acc * alpha
    if bias is not None:
        acc += bias[:N].float()
    if rowvec is not None:
        acc = (acc.view(Bo, Ho * Wo, N) + rowvec[:, :N].float().unsqueeze(1)).reshape(M, N)
    if residual is not None:
        acc += residual.float().reshape(M, N)
    if act == 1:
        acc = torch.nn.functional.silu(acc)
    if out.dtype == torch.float32 and round_bf16:
        acc = acc.to(BF16).float()
    out.copy_(acc.view(out.shape).to(out.dtype))
    return out


def interp_wgrad_any(p_src, q_src, out, *, lin, M, os_row, os_col, alpha=1.0, q_c0=0, taps=((0, 0),),
                     tap_off=(0,), **kw):
    w = min(64, q_src.C - q_c0)
    assert w > 0 and w % 8 == 0, (q_src.C, q_c0)
    if RECORD is not None:
        RECORD.append(("wgrad", dict(q_C=q_src.C, q_c0=q_c0, width=w, out=out, os_row=os_row, os_col=os_col)))
    if lin:
        rows = min(M, p_src.W, q_src.W)
        P = mat(p_src.ptr, rows, p_src.C, p_src.sW).float()
        Q = mat(q_src.ptr, rows, q_src.C, q_src.sW)[:, q_c0:q_c0 + w].float()
        o = out.as_strided((P.shape[1], w), (os_row, os_col), out.storage_offset() + tap_off[0])
        o += alpha * (P.t() @ Q)
        return out
    Wo, Ho = kw["geo"]
    Bo = M // (Wo * Ho)
    Q = a_nhwc(q_src).float().reshape(-1, q_src.C)[:M, q_c0:q_c0 + w]
    for (dw, dh), off in zip(taps, tap_off):
        P = shifted_rows(p_src, dw, dh, Wo, Ho, Bo)
        o = out.as_strided((P.shape[1], w), (os_row, os_col), out.storage_offset() + off)
        o += alpha * (P.t() @ Q)
    return out


class RankCalls(ops_interp.PcmCalls):
    def pcm_lora_refresh(self, master, table, num_entries, total_work, scale, opnd):
        """Any-rank lora_refresh_kernel: per entry ceil(r/64) * (taps*cin/64 + cout/64) tiles."""
        _raw = ops_interp._raw
        import ctypes
        tab = _raw(table, num_entries * 9, ctypes.c_int64, torch.int64).view(num_entries, 9).tolist()
        work = 0
        for a_off, b_off, a_fwd, sb_fwd, sb_t, a_t, ci, co, w0 in tab:
            cin, taps, cout, r = ci & 0xffffffff, ci >> 32, co & 0xffffffff, co >> 32
            assert w0 == work
            k = taps * cin
            A = _raw(master + 4 * a_off, r * k, ctypes.c_float, torch.float32).view(r, k).to(BF16)
            sB = (_raw(master + 4 * b_off, cout * r, ctypes.c_float, torch.float32).view(cout, r) * scale).to(BF16)
            o = lambda off, n: _raw(opnd + 2 * off, n, ctypes.c_uint16, torch.int16).view(BF16)  # noqa: E731
            o(a_fwd, r * k).view(r, k).copy_(A)
            o(a_t, r * k).view(cin, taps * r).copy_(A.view(r, taps, cin).permute(2, 1, 0).reshape(cin, taps * r))
            o(sb_fwd, cout * r).view(cout, r).copy_(sB)
            o(sb_t, cout * r).view(r, cout).copy_(sB.t())
            work += math.ceil(r / 64) * (k // 64 + cout // 64)
        assert work == total_work


def _install(monkeypatch, step=False):
    from pcm_b200 import ops
    ops_interp.install(monkeypatch)
    monkeypatch.setattr(ops, "gemm", interp_gemm_any)
    monkeypatch.setattr(ops, "wgrad", interp_wgrad_any)
    if step:
        monkeypatch.setattr(ops, "_call", RankCalls())


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _build(cfg, P, **kw):
    from pcm_b200 import ops
    from pcm_b200.unet import UNetB200
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        net = UNetB200(cfg, P, "cpu", lora=True, need_backward=True, **kw)
    finally:
        ops.DRY_RUN = old
    refresh_operands(net)
    return net


def _setup(cfg_name, r, B=2, hw=8, seed=0):
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config
    ocfg = dataclasses.replace(getattr(unet_ref, cfg_name), lora_rank=r)
    P = unet_ref.init_params(ocfg, seed, lora_b_std=0.02)
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=seed)
    net = _build(dataclasses.replace(getattr(config, cfg_name), lora_rank=r), P)
    return ocfg, P, batch, net


# ------------------------------------------------------------------------------------------------
# the contract
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [4, 12, 264, 0, 100])
def test_unsupported_ranks_raise(r):
    from pcm_b200 import config, weights
    from pcm_b200.unet import UNetB200
    cfg = dataclasses.replace(config.TINY, lora_rank=r)
    with pytest.raises(ValueError, match="supported ranks"):
        config.check_lora_rank(r)
    sd = weights.synthetic_state_dict(dataclasses.replace(config.TINY, lora_rank=64), 0)
    with pytest.raises(ValueError, match="supported ranks"):
        UNetB200(cfg, sd, "cpu", lora=True, need_backward=True)


def test_rank_mismatched_state_dict_raises():
    from pcm_b200 import config, ops, weights
    from pcm_b200.unet import UNetB200
    sd = weights.synthetic_state_dict(dataclasses.replace(config.TINY, lora_rank=32), 0)
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        with pytest.raises(ValueError, match=r"rank-32 .* rank 16"):
            UNetB200(dataclasses.replace(config.TINY, lora_rank=16), sd, "cpu", lora=True, need_backward=True)
    finally:
        ops.DRY_RUN = old


@pytest.mark.parametrize("mod", ["train_pcm_lora_sd15", "train_pcm_lora_sdxl_adv"])
def test_cli_lora_rank(mod):
    import importlib
    m = importlib.import_module("pcm_b200." + mod)
    base = ["--synthetic", "--max_train_steps", "1"] + (["--adv_weight", "0"] if "sdxl" in mod else [])
    assert m.parse_args(base).lora_rank == 64
    for r in (8, 32, 48, 128, 256):
        assert m.parse_args(base + ["--lora_rank", str(r)]).lora_rank == r
    for r in (4, 12, 264):
        with pytest.raises(ValueError, match="supported ranks"):
            m.parse_args(base + ["--lora_rank", str(r)])


# ------------------------------------------------------------------------------------------------
# the launch plans
# ------------------------------------------------------------------------------------------------
def _record_step(monkeypatch, cfg_name, r, B=2, hw=8):
    global RECORD
    ocfg, P, batch, net = _setup(cfg_name, r, B, hw)
    _install(monkeypatch)
    x, ctx = batch["latents"], batch["prompt_embeds"]
    added = (batch["text_embeds"], batch["time_ids"]) if getattr(ocfg, "addition_embed", False) else None
    RECORD = []
    try:
        net.forward(_nhwc(x), torch.tensor([999, 19])[:B], ctx.to(BF16).reshape(B * ctx.shape[1], -1),
                    lora=True, save=True, added_cond=added, lora_batch=1)
        net.lora_grad.zero_()
        net.backward(torch.randn(1, hw, hw, 4) * 1e-3)
        return net, RECORD
    finally:
        RECORD = None


@pytest.mark.parametrize("r", [8, 32, 48, 64, 96, 128, 256])
def test_plan_chunk_and_slice_widths(monkeypatch, r):
    """Every LoRA K entry (an operand of extent r) multiplies r columns in ceil(r/64) chunks, every
    weight-gradient slice stays inside the layer's ranks and the slices of one output cover them once;
    at r = 64 every width is 64."""
    net, rec = _record_step(monkeypatch, "TINY", r)
    gemms = [info for kind, info in rec if kind == "gemm"]
    narrow = [info for info in gemms if sum(info["widths"]) != 64 * len(info["widths"])]
    # a LoRA entry (rank-side operand of extent r): ceil(r/64) chunks, r columns in all
    lora = [info for info in gemms if info["a_C"] % r == 0 and info["b_K"] % r == 0
            and (info["a_C"] == r or info["b_K"] == r)]
    assert lora and all(len(i["widths"]) == math.ceil(r / 64) and sum(i["widths"]) == r for i in lora)
    assert (len(narrow) > 0) == (r % 64 != 0) and all(i in lora for i in narrow)
    if r == 64:
        assert all(w == 64 for info in gemms for w in info["widths"])
    wg = [info for kind, info in rec if kind == "wgrad"]
    for info in wg:
        assert info["width"] <= 64 and info["q_c0"] + info["width"] <= info["q_C"]
        if r % 64:
            assert info["q_C"] - info["q_c0"] <= r, info    # the view ends at the layer's last rank
    # the slices of one gradient launch group cover the layer's r ranks once: widths add up to r per
    # ceil(r/64) consecutive launches into the same gradient rows
    for L in net.lora_layers:
        assert L.lora.gA.shape[0] == r and L.lora.gB.shape[1] == r
    assert sum(i["width"] for i in wg) % r == 0 and len(wg) % math.ceil(r / 64) == 0


@pytest.mark.parametrize("r", [8, 32, 48, 128, 256])
def test_forward_and_backward_match_the_oracle_tiny(monkeypatch, r):
    _fwd_bwd(monkeypatch, "TINY", r)


@pytest.mark.parametrize("r", [8, 48, 128])
def test_forward_and_backward_match_the_oracle_tiny_xl(monkeypatch, r):
    _fwd_bwd(monkeypatch, "TINY_XL", r)


def _fwd_bwd(monkeypatch, cfg_name, r):
    from oracle import unet_ref
    B, hw = 2, 8
    ocfg, P, batch, net = _setup(cfg_name, r, B, hw)
    _install(monkeypatch)
    x, ctx = batch["latents"], batch["prompt_embeds"]
    ts = torch.tensor([999, 19])
    okw, added = {}, None
    if getattr(ocfg, "addition_embed", False):
        added = (batch["text_embeds"], batch["time_ids"])
        okw = dict(added_cond_kwargs=dict(text_embeds=batch["text_embeds"], time_ids=batch["time_ids"]))
    ctx2 = ctx.to(BF16).reshape(B * ctx.shape[1], -1)
    ref = unet_ref.UNetRef(ocfg, P, use_lora=True, emulate_bf16=True)(x, ts, ctx, **okw)
    out = _nchw(net.forward(_nhwc(x), ts, ctx2, lora=True, added_cond=added))
    err = (out - ref).abs()
    assert err.max().item() <= 3e-2 * ref.abs().max().item(), err.max().item()
    assert err.mean().item() <= 1e-2 * ref.pow(2).mean().sqrt().item(), err.mean().item()
    G = torch.randn(B, 4, hw, hw, generator=torch.Generator().manual_seed(7)) / (B * 4 * hw * hw)
    Pg = {k: (v.clone().requires_grad_(True) if ".lora_" in k else v) for k, v in P.items()}
    eps = unet_ref.UNetRef(ocfg, Pg, use_lora=True, emulate_bf16=True)(x, ts, ctx, **okw)
    (eps * G).sum().backward()
    net.forward(_nhwc(x), ts, ctx2, lora=True, save=True, added_cond=added)
    net.lora_grad.zero_()
    net.backward(_nhwc(G))
    g = net.lora_grad_dict()
    num = den = 0.0
    for k, v in Pg.items():
        if ".lora_" in k:
            assert g[k].shape[0 if "lora_A" in k else 1] == r
            num += (g[k].float() - v.grad.reshape(g[k].shape)).pow(2).sum().item()
            den += v.grad.pow(2).sum().item()
    assert (num / den) ** 0.5 <= 5e-2, (num / den) ** 0.5


@pytest.mark.parametrize("cfg_name,r", [("TINY", 8), ("TINY", 48), ("TINY", 128), ("TINY_XL", 48)])
def test_step_matches_the_oracle_iteration(monkeypatch, cfg_name, r):
    """PCMTrainStep.forward_backward on CPU at rank r vs oracle/pcm_ref.pcm_step_ref."""
    from oracle import pcm_ref, unet_ref
    from pcm_b200 import config, ops
    from pcm_b200.step import PCMTrainStep
    B, hw, mp = 2, 8, 4
    xl = cfg_name == "TINY_XL"
    ocfg = dataclasses.replace(getattr(unet_ref, cfg_name), lora_rank=r)
    P = unet_ref.init_params(ocfg, 0, lora_b_std=0.02)
    nd = 40 if xl else 50
    batch = pcm_ref.make_batch(ocfg, B, hw, seed=0, num_ddim=nd, **(dict(zero_uncond=True) if xl else {}))
    ref = pcm_ref.pcm_step_ref(ocfg, P, batch, multiphase=mp, num_ddim=nd, emulate_bf16=True, need_grad=not xl)
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        st = PCMTrainStep(dataclasses.replace(getattr(config, cfg_name), lora_rank=r), P, "cpu", batch=B,
                          height=hw, width=hw, multiphase=mp, num_ddim_timesteps=nd, keep_debug=True)
    finally:
        ops.DRY_RUN = old
    net = st.unet
    _install(monkeypatch, step=True)
    net.refresh_lora()          # the any-rank refresh table through its interpreter
    extra = dict(text_embeds=batch["text_embeds"].to(BF16), time_ids=batch["time_ids"]) if xl else {}
    st.load_inputs(_nhwc(batch["latents"]), _nhwc(batch["noise"]), batch["index"], batch["w"],
                   batch["prompt_embeds"].to(BF16), batch["uncond_prompt_embeds"].to(BF16), **extra)
    net.lora_grad.zero_()
    st.forward_backward()
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()  # noqa: E731
    assert rel(_nchw(st.x_prev), ref["x_prev"]) < 2e-2 and rel(_nchw(st.model_pred), ref["model_pred"]) < 2e-2
    assert abs(st.loss.item() - ref["loss"].item()) <= 4e-2 * ref["loss"].item()
    if xl:
        assert net.lora_grad.abs().max() > 0
        return
    g = net.lora_grad_dict()
    dot = n1 = n2 = 0.0
    for k, rg in ref["grads"].items():
        gg = g[k].float().reshape(rg.shape)
        dot += (gg * rg).sum().item()
        n1 += gg.pow(2).sum().item()
        n2 += rg.pow(2).sum().item()
    assert dot / (n1 ** 0.5 * n2 ** 0.5) >= 0.85


@pytest.mark.parametrize("r", [8, 48, 128])
def test_refresh_table_writes_the_layer_views(monkeypatch, r):
    """The refresh table (interpreted like lora_refresh_kernel) writes exactly the per-layer operand views."""
    from pcm_b200 import config, ops, weights
    cfg = dataclasses.replace(config.TINY, lora_rank=r)
    sd = weights.synthetic_state_dict(cfg, 0, lora_b_std=0.2)
    net = _build(cfg, sd)
    want = net.lora_opnd.clone()
    net.lora_opnd.fill_(float("nan"))
    monkeypatch.setattr(ops, "_call", RankCalls())
    net.refresh_lora()
    assert torch.equal(net.lora_opnd, want)
    assert net.refresh_work == sum(math.ceil(r / 64) * ((L.k * L.k if L.kind == "conv" else 1) * L.cin // 64
                                                        + L.cout // 64) for L in net.lora_layers)
