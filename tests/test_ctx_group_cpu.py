"""Cross-attention k / v of all transformer blocks as context chunks (UNetB200.ctx_kv_all): the HOST side
of that plan - stacked operand layout, chunking, K programs, column windows - checked on CPU by
interpreting the recorded `pcm_gemm` descriptors with torch (a test-side interpreter of the K-program
semantics in include/pcm_b200.h; the product never computes on the CPU) and comparing every block's k / v
with the per-layer definition  y = x W^T + s (x A^T) B^T  (peft LoRA Linear, SURVEY.md section 8 row U).

The interpreter reads the operands through the raw pointers of the descriptors, exactly what the CUDA side
gets, so a wrong offset / stride / row range in the plan shows up here."""
import pytest
import torch

from gemm_interp import BF16, build_net, interp_gemm as _interp_gemm


@pytest.mark.parametrize("cfg_name", ["TINY", "TINY_XL"])
@pytest.mark.parametrize("lora_rows", [None, 1])
def test_context_chunks_match_per_layer_projections(monkeypatch, cfg_name, lora_rows):
    from pcm_b200 import config, ops
    from pcm_b200.unet import UNetB200, _Pass
    cfg = getattr(config, cfg_name)
    net, sd = build_net(cfg)
    assert net.ctx_group is not None and len(net.ctx_group.chunks) >= 1
    r, s = net.r, net.scale
    B, S = 3, 77
    ctx = torch.randn(B * S, cfg.cross_attention_dim, generator=torch.Generator().manual_seed(5)).to(BF16)
    Ml = (lora_rows or B) * S
    monkeypatch.setattr(ops, "gemm", _interp_gemm)
    kv = net.ctx_kv_all(_Pass(lora=True, B=B, lb=lora_rows or B, ctx=ctx))
    blocks = [n[:-len(".attn2.to_k")] for n in net._ctx_names if n.endswith(".attn2.to_k")]
    assert sorted(kv) == sorted(blocks)
    seen_windows = set()
    for t in blocks:
        k, v, T = kv[t]
        assert T.shape == (Ml, 2 * r) and k.shape[0] == B * S
        assert v.storage_offset() == k.storage_offset() + k.shape[1] and v.stride(0) == k.stride(0)
        seen_windows.add((k.untyped_storage().data_ptr(), k.storage_offset() % k.stride(0)))
        for i, (suf, got) in enumerate(((".attn2.to_k", k), (".attn2.to_v", v))):
            W = sd[t + suf + ".weight"].to(BF16).float()
            A = sd[t + suf + ".lora_A.weight"].to(BF16).float()
            sB = (s * sd[t + suf + ".lora_B.weight"]).to(BF16).float()
            x = ctx.float()
            Tref = (x[:Ml] @ A.t()).to(BF16)
            assert torch.equal(T[:, i * r:(i + 1) * r], Tref), (t, suf)
            ref = x @ W.t()
            ref[:Ml] += Tref.float() @ sB.t()
            err = (got.float() - ref).abs().max().item()
            assert err <= 2e-2 * ref.abs().max().item() + 1e-3, (t, suf, err)
            # the LoRA term is really there (and only on the leading rows)
            base = (x @ W.t())
            d = (got.float() - base).abs()
            assert Ml == B * S or d[:Ml].max() > 5 * d[Ml:].max()
    assert len(seen_windows) == len(blocks)       # every block has its own column window
    # the leading rows, as the target pass takes them
    rows = S
    sub = UNetB200.ctx_kv_rows(kv, rows)
    for t in blocks:
        assert sub[t][2] is None and torch.equal(sub[t][0], kv[t][0][:rows]) and torch.equal(sub[t][1], kv[t][1][:rows])


def test_context_chunks_respect_the_k_program_limit():
    """SDXL: 70 transformer blocks -> chunks of <= 11 blocks of one width; N ranges aligned to block_n."""
    from pcm_b200 import _lib, config
    from oracle.unet_ref import layer_table
    tab = layer_table(config.SDXL)
    names = [n for n, *_ in tab if n.endswith(".attn2.to_k")]
    assert len(names) == 70
    # replicate the chunking rule on the table (no 2.6 G-parameter network is built here)
    co = {n: c for n, _, _, c, _ in tab}
    names.sort(key=lambda n: co[n])
    chunks, cur = [], None
    for n in names:
        if cur is None or cur[0] != co[n] or len(cur[1]) == 11:
            cur = (co[n], [])
            chunks.append(cur)
        cur[1].append(n)
    assert [len(c[1]) for c in chunks] == [10, 11, 11, 11, 11, 11, 5]
    for c, blk in chunks:
        assert 1 + 2 * len(blk) <= _lib.MAX_PROG and 2 * c * len(blk) < 65536 and c % 160 == 0
