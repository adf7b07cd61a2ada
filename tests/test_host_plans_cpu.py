"""HOST launch plans of the LoRA-fused Linear layers, checked on CPU by interpreting the `pcm_gemm`
descriptors they build (tests/gemm_interp.py) against the peft definition
    y = x W^T + b + s (x A^T) B^T
(SURVEY.md section 8 row U; train_pcm_lora_sd15.py:868-885 wraps these modules with get_peft_model).

Covers the plans the CUDA kernels cannot check by themselves: which stacked operand rows / columns a
layer's LoRA K block reads, the N ranges of grouped layers, the adapter-on-leading-rows layout of the merged
student + teacher pass, the residual / bias epilogue arguments.  (The kernels behind the same descriptors are
compared with torch on the GPU in tests/test_gemm_gpu.py; the whole network against the oracle in
tests/test_unet_gpu.py and tests/test_parity_gpu.py.)"""
import pytest
import torch

from gemm_interp import BF16, build_net, interp_gemm, interp_wgrad as interp_wgrad_, lora_linear_ref
from pcm_b200.unet import _Backward, _Pass


@pytest.fixture(scope="module")
def tiny():
    from pcm_b200 import config
    return build_net(config.TINY)


def _close(got, ref, what):
    err = (got.float() - ref).abs().max().item()
    assert err <= 1.2e-2 * ref.abs().max().item() + 1e-3, (what, err)


def _x(rows, cols, seed):
    return torch.randn(rows, cols, generator=torch.Generator().manual_seed(seed)).to(BF16)


@pytest.mark.parametrize("lora_rows", [None, 128])
def test_linear_fuses_lora_residual_and_bias_on_the_pass_rows(monkeypatch, tiny, lora_rows):
    """attn1.to_out.0 (bias, residual) and ff.net.2: T = x A^T as its own launch on the adapter rows, then
    one GEMM with the LoRA block as an extra K entry."""
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    M = 384
    P = _Pass(lora=True, B=M, lb=lora_rows or M)
    for name in ("down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_out.0",
                 "down_blocks.1.attentions.1.transformer_blocks.0.ff.net.2",
                 "mid_block.attentions.0.proj_in"):
        L = net.layers[name]
        x, res = _x(M, L.cin, 1), _x(M, L.cout, 2)
        tape = []
        y = net.linear(P, name, [x], residual=res, save=tape)
        ref = lora_linear_ref(sd, name, x, net.scale, lora_rows) + res.float()
        _close(y, ref, name)
        (_, nm, xs, T), = tape
        assert nm == name and T.shape == ((lora_rows or M), net.r) and xs[0].shape[0] == (lora_rows or M)
        # without the adapter: the frozen layer
        y0 = net.linear(_Pass(lora=False, B=M, lb=M), name, [x])
        W = sd[name + ".weight"].reshape(L.cout, -1).to(BF16).float()
        _close(y0, x.float() @ W.t() + sd[name + ".bias"].float(), name + " base")
        assert (y.float() - res.float() - y0.float())[: (lora_rows or M)].abs().max() > 1e-2   # the adapter is live


def test_linear_reads_channel_concatenated_sources(monkeypatch, tiny):
    """conv_shortcut of an up-block resnet: two A sources (hidden state, skip) = torch.cat along channels."""
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    name = "up_blocks.1.resnets.0.conv_shortcut"
    L = net.layers[name]
    c1 = L.cin // 2
    M = 256
    xa, xb = _x(M, c1, 3), _x(M, L.cin - c1, 4)
    y = net.linear(_Pass(lora=True, B=M, lb=M), name, [xa, xb])
    _close(y, lora_linear_ref(sd, name, torch.cat([xa, xb], 1), net.scale), name)


@pytest.mark.parametrize("lora_rows", [None, 128])
def test_qkv_group_equals_three_lora_linears(monkeypatch, tiny, lora_rows):
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    t = "down_blocks.1.attentions.0.transformer_blocks.0"
    G = net.groups[t + ".attn1.to_q"]
    M = 384
    x = _x(M, G.cin, 7)
    tape = []
    q, k, v = net.linear_group(_Pass(lora=True, B=M, lb=lora_rows or M), t + ".attn1.to_q", x, save=tape)
    for suf, got in ((".attn1.to_q", q), (".attn1.to_k", k), (".attn1.to_v", v)):
        _close(got, lora_linear_ref(sd, t + suf, x, net.scale, lora_rows), t + suf)
    assert q.stride(0) == 3 * G.cout and tape[0][3].shape == ((lora_rows or M), 3 * net.r)


@pytest.mark.parametrize("lora_rows", [None, 1])
def test_time_embedding_projections_run_as_one_group(monkeypatch, tiny, lora_rows):
    """All resnets' time_emb_proj(silu(temb)) from ONE grouped launch: column range i == layer i."""
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    G = net.temb_group
    assert G is not None and G.g == len([n for n in net.layers if n.endswith(".time_emb_proj")])
    B = 3
    st = _x(B, G.cin, 9)
    out, T = net.temb_all(_Pass(lora=True, B=B, lb=lora_rows or B, st=st))
    assert T.shape == ((lora_rows or B), G.g * net.r)
    for i, name in enumerate(G.names):
        _close(out[:, G.offs[i]:G.offs[i + 1]], lora_linear_ref(sd, name, st, net.scale, lora_rows), name)


def test_forward_operands_equal_the_state_dict(tiny):
    """Every forward operand the plans read (K-blocked, single or stacked) is the state-dict tensors of its
    member layers in bf16, OHWI for convolutions, each member at its first row."""
    from gemm_interp import b_matrix
    from pcm_b200 import ops
    net, sd = tiny
    checked = 0
    for key, op in net.operands.items():
        rows = [sd[L.name + ".weight"] for L, _ in op.members]
        Wg = torch.cat([W.permute(0, 2, 3, 1).reshape(W.shape[0], -1) if W.dim() == 4 else W for W in rows]).to(BF16)
        assert torch.equal(b_matrix(ops.bsrc(op.w)), Wg), key
        assert [n0 for _, n0 in op.members] == [sum(W.shape[0] for W in rows[:i]) for i in range(len(rows))], key
        checked += 1
    assert checked > 40


@pytest.mark.parametrize("cfg_name", ["TINY", "TINY_XL"])
def test_each_frozen_weight_is_held_by_one_forward_operand(cfg_name):
    """Every frozen Linear / conv weight of the layer table is held by exactly one forward operand, in a
    storage of its own, and the operands hold exactly the table's forward-weight bytes: teacher, student and
    target share that single copy.  No other bf16 copy of a forward weight is reachable from the layers or
    groups (besides the dgrad operands and conv_in, whose 4-channel kernel reads its own layout)."""
    import types
    from pcm_b200 import config
    from pcm_b200.unet import _Layer, _Lora
    cfg = getattr(config, cfg_name)
    net, _ = build_net(cfg)
    want = {n: 2 * cout * k * k * cin if kind == "conv" else 2 * cout * cin
            for n, kind, cin, cout, k in config.layer_table(cfg) if kind not in ("gn", "ln") and n != "conv_in"}
    held = sorted(L.name for op in net.operands.values() for L, _ in op.members)
    assert held == sorted(want)
    storages = {op.w.untyped_storage().data_ptr() for op in net.operands.values()}
    assert len(storages) == len(net.operands)
    assert sum(op.w.untyped_storage().nbytes() for op in net.operands.values()) == sum(want.values())

    def reach(obj, path, out):
        if isinstance(obj, torch.Tensor):
            if obj.dtype == BF16:
                out.append((path, obj))
        elif isinstance(obj, (list, tuple)):
            for i, v in enumerate(obj):
                reach(v, f"{path}[{i}]", out)
        elif isinstance(obj, dict):
            for k, v in obj.items():
                reach(v, f"{path}[{k!r}]", out)
        elif isinstance(obj, (_Layer, _Lora)):
            for s in type(obj).__slots__:
                reach(getattr(obj, s, None), f"{path}.{s}", out)
        elif isinstance(obj, types.SimpleNamespace):
            for k, v in vars(obj).items():
                if k not in ("layers", "blocks"):           # reached through net.layers / net.groups
                    reach(v, f"{path}.{k}", out)
        return out

    tensors = reach([net.layers, net.groups, net.temb_group, net.ctx_group], "net", [])
    assert any(p.endswith(".w_t_cat") for p, _ in tensors) and any(".lora." in p for p, _ in tensors)
    allowed = storages | {net.lora_opnd.untyped_storage().data_ptr()}
    for path, t in tensors:
        if path.rsplit(".", 1)[-1] in ("w_t", "w_t_cat", "w_c4", "w_c4_t"):
            continue
        assert t.untyped_storage().data_ptr() in allowed, path


def _autograd_ref(sd, names, x, dys, scale, lora_rows):
    """float64 autograd through  y_i = x W_i^T + s (x A_i^T) B_i^T  (bf16-rounded parameters; adapter on
    the leading rows): returns dx and {name: (dA, dB)}."""
    x64 = x.double().requires_grad_(True)
    params, loss = {}, 0.0
    rows = x.shape[0] if lora_rows is None else lora_rows
    for name, dy in zip(names, dys):
        W = sd[name + ".weight"]
        W = W.reshape(W.shape[0], -1).to(BF16).double()
        A = sd[name + ".lora_A.weight"]
        A = A.reshape(A.shape[0], -1).to(BF16).double().requires_grad_(True)
        Bm = sd[name + ".lora_B.weight"]
        Bm = Bm.reshape(Bm.shape[0], -1).to(BF16).double().requires_grad_(True)
        y = x64 @ W.t()
        y = torch.cat([y[:rows] + scale * (x64[:rows] @ A.t()) @ Bm.t(), y[rows:]], 0)
        loss = loss + (y[:dy.shape[0]] * dy.double()).sum()
        params[name] = (A, Bm)
    loss.backward()
    return x64.grad, {n: (a.grad, b.grad) for n, (a, b) in params.items()}


def _rel(got, ref):
    return ((got.double() - ref).norm() / (ref.norm() + 1e-30)).item()


def test_linear_backward_launch_plan(monkeypatch, tiny):
    """linear_bwd: dt = dy (sB), dx = [dy | dt] [W ; A], and the two LoRA weight-gradient launches land in the
    layer's slices of the flat gradient buffer."""
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    monkeypatch.setattr(ops, "wgrad", interp_wgrad_)
    name = "down_blocks.1.attentions.1.transformer_blocks.0.ff.net.2"
    L = net.layers[name]
    M = 256
    x, dy = _x(M, L.cin, 11), _x(M, L.cout, 12)
    tape = []
    net.linear(_Pass(lora=True, B=M, lb=M), name, [x], save=tape)
    net.lora_grad.zero_()
    dx = net.linear_bwd(_Backward(), tape[0], dy)
    dx_ref, g = _autograd_ref(sd, [name], x, [dy], net.scale, None)
    assert _rel(dx, dx_ref) < 1e-2
    dA, dB = g[name]
    assert _rel(L.lora.gA, dA) < 1e-2 and _rel(L.lora.gB, dB) < 1e-2
    # nothing outside this layer's slices of the flat buffer was touched
    lo = L.lora
    mask = torch.ones_like(net.lora_grad, dtype=torch.bool)
    mask[lo.a_off:lo.a_off + lo.gA.numel()] = False
    mask[lo.b_off:lo.b_off + lo.gB.numel()] = False
    assert not net.lora_grad[mask].any()


@pytest.mark.parametrize("lead,need_dx", [(".attn1.to_q", True), (".attn2.to_k", False)])
def test_grouped_backward_launch_plan(monkeypatch, tiny, lead, need_dx):
    """linear_group_bwd over the packed output gradients [dq | dk | dv] (resp. [dk | dv], no input gradient:
    the text context is not trained), with T a column window of a wider stacked down-projection."""
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    monkeypatch.setattr(ops, "wgrad", interp_wgrad_)
    t = "down_blocks.1.attentions.0.transformer_blocks.0"
    G = net.groups[t + lead]
    M = 154 if not need_dx else 256
    x = _x(M, G.cin, 13)
    P = _Pass(lora=True, B=M, lb=M, ctx=x)
    dys = [_x(M, G.cout, 20 + i) for i in range(G.g)]
    dpk = torch.cat(dys, 1).contiguous()
    if need_dx:
        tape = []
        net.linear_group(P, t + lead, x, save=tape)
        rec = tape[0]
    else:
        kv = net.ctx_kv_all(P)                  # T = this block's window of the stacked context projection
        rec = ("lgroup", t + lead, x, kv[t][2])
        assert rec[3].stride(0) == net.ctx_group.nl * net.r
    net.lora_grad.zero_()
    dx = net.linear_group_bwd(_Backward(), rec, dpk, need_dx=need_dx)
    dx_ref, g = _autograd_ref(sd, G.names, x, dys, net.scale, None)
    if need_dx:
        assert _rel(dx, dx_ref) < 1e-2
    else:
        assert dx is None
    for n in G.names:
        lo = net.layers[n].lora
        assert _rel(lo.gA, g[n][0]) < 1e-2 and _rel(lo.gB, g[n][1]) < 1e-2, n


# ---------------------------------------------------------------------------------------------
# 3x3 convolutions: implicit-GEMM K programs (taps, skip concat, stride-2 parity planes) + LoRA
# ---------------------------------------------------------------------------------------------
def _conv_ref(sd, name, x_nchw, scale, stride, lora_samples=None, dtype=torch.float64):
    """peft LoRA Conv2d on bf16-rounded parameters: conv(x, W) + b + s * B(A(x)), A = k x k conv with the
    layer's stride / padding, B = 1x1 (SURVEY.md section 8c); adapter on the leading samples only."""
    F = torch.nn.functional
    W = sd[name + ".weight"].to(BF16).to(dtype)
    b = sd[name + ".bias"].to(dtype)
    A = sd[name + ".lora_A.weight"].to(BF16).to(dtype)
    Bm = sd[name + ".lora_B.weight"].to(BF16).to(dtype)
    y = F.conv2d(x_nchw, W, b, stride=stride, padding=1)
    n = x_nchw.shape[0] if lora_samples is None else lora_samples
    ad = scale * F.conv2d(F.conv2d(x_nchw[:n], A, None, stride=stride, padding=1), Bm)
    return torch.cat([y[:n] + ad, y[n:]], 0), (A, Bm)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _img(b, c, h, w, seed):
    return torch.randn(b, c, h, w, generator=torch.Generator().manual_seed(seed)).to(BF16)


@pytest.mark.parametrize("lora_samples", [None, 1])
def test_resnet_conv_reads_skip_concat_row_vector_and_residual(monkeypatch, tiny, lora_samples):
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    name = "up_blocks.1.resnets.0.conv1"          # input = cat(hidden, skip)
    L = net.layers[name]
    B, H, W = 3, 8, 8
    c1 = L.cin // 2
    xa, xb = _img(B, c1, H, W, 31), _img(B, L.cin - c1, H, W, 32)
    rv = _x(B, L.cout, 33)
    res = _img(B, L.cout, H, W, 34)
    tape = []
    y = net.conv3(_Pass(lora=True, B=B, lb=lora_samples or B), name, [_nhwc(xa), _nhwc(xb)], rowvec=rv,
                  residual=_nhwc(res), save=tape)
    ref, _ = _conv_ref(sd, name, torch.cat([xa, xb], 1).double(), net.scale, 1, lora_samples)
    ref = ref + rv.double()[:, :, None, None] + res.double()
    assert _rel(y.permute(0, 3, 1, 2), ref) < 6e-3
    assert tape[0][3].shape == ((lora_samples or B), H, W, net.r)


def test_downsample_conv_reads_four_parity_planes(monkeypatch, tiny):
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    name = "down_blocks.0.downsamplers.0.conv"
    L = net.layers[name]
    B, H, W = 2, 8, 8
    x = _img(B, L.cin, H, W, 35)
    y = net.conv3(_Pass(lora=True, B=B, lb=B), name, [_nhwc(x)], stride=2)
    ref, _ = _conv_ref(sd, name, x.double(), net.scale, 2)
    assert y.shape == (B, H // 2, W // 2, L.cout) and _rel(y.permute(0, 3, 1, 2), ref) < 6e-3


@pytest.mark.parametrize("name,stride", [("down_blocks.1.resnets.0.conv2", 1), ("down_blocks.0.downsamplers.0.conv", 2)])
def test_conv_backward_launch_plan(monkeypatch, tiny, name, stride):
    """conv3_bwd: dgrad over flipped taps (stride 2: one launch per parity plane of dx, written through a
    strided view), dt = dy (sB), and the tap-wise LoRA weight gradients - against float64 autograd."""
    from pcm_b200 import ops
    net, sd = tiny
    monkeypatch.setattr(ops, "gemm", interp_gemm)
    monkeypatch.setattr(ops, "wgrad", interp_wgrad_)
    L = net.layers[name]
    B, H, W = 2, 8, 8
    x = _img(B, L.cin, H, W, 41)
    dy = _img(B, L.cout, H // stride, W // stride, 42)
    tape = []
    net.conv3(_Pass(lora=True, B=B, lb=B), name, [_nhwc(x)], stride=stride, save=tape)
    net.lora_grad.zero_()
    dx = net.conv3_bwd(_Backward(), tape[0], _nhwc(dy))
    x64 = x.double().requires_grad_(True)
    F = torch.nn.functional
    Wt = sd[name + ".weight"].to(BF16).double()
    A = sd[name + ".lora_A.weight"].to(BF16).double().requires_grad_(True)
    Bm = sd[name + ".lora_B.weight"].to(BF16).double().requires_grad_(True)
    y = (F.conv2d(x64, Wt, None, stride=stride, padding=1) +
         net.scale * F.conv2d(F.conv2d(x64, A, None, stride=stride, padding=1), Bm))
    (y * dy.double()).sum().backward()
    assert _rel(dx.permute(0, 3, 1, 2), x64.grad) < 1e-2
    lo = L.lora
    gA = lo.gA.view(net.r, 3, 3, L.cin).permute(0, 3, 1, 2)        # [r, (kh, kw, cin)] -> [r, cin, kh, kw]
    assert _rel(gA, A.grad) < 1e-2
    assert _rel(lo.gB, Bm.grad.reshape(L.cout, net.r)) < 1e-2


def test_refresh_table_writes_exactly_the_per_layer_operand_views(tiny):
    """`pcm_lora_refresh` is driven by an offset table; the GEMM plans read the operand buffer through
    per-layer and stacked views.  Interpreting the table must reproduce the view-based fill bit for bit
    and leave no element of the buffer unwritten."""
    from ops_interp import PcmCalls
    from gemm_interp import refresh_operands
    net, _ = tiny
    want = net.lora_opnd.clone()
    net.lora_opnd.view(torch.int16).fill_(0x7fc1)            # a NaN pattern no refresh writes
    PcmCalls().pcm_lora_refresh(net.lora_master.data_ptr(), net.refresh_table.data_ptr(),
                                net.refresh_table.shape[0], net.refresh_work, net.scale, net.lora_opnd.data_ptr())
    got = net.lora_opnd.clone()
    assert not (got.view(torch.int16) == 0x7fc1).any()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    refresh_operands(net)
    assert torch.equal(net.lora_opnd.view(torch.int16), want.view(torch.int16))
