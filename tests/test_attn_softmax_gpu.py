"""The forward's online-softmax paths: full 64-key blocks (no key mask), the masked last block of a
ragged Skv, and the O rescale that is skipped when no row of a warp has a new maximum.  The logits
follow a trend along the keys, one 64-key block apart by STEP: rising, every block raises every row's
maximum (alpha < 1 at each block); falling, block 0 holds every row's maximum (alpha = 1 from block 1
on, so the rescale is always skipped).  Head sizes cover the trimmed d <= 40 products, the 64-column
block and two blocks (d = 80).  Every case must match float64 as tests/test_attn_gpu.py requires
(same check, same NaN-guarded layouts); the inputs are checked to have the trend they claim."""
import pytest
import torch

import test_attn_gpu
from test_attn_gpu import BF, _case_id, _sweep_case, check_case

pytestmark = pytest.mark.gpu

STEP = 16.0   # logit change per 64 keys; the other head coordinates add logits of std ~1/4

# Skv: a multiple of 64 (no masked block), ragged (77: one full block and a masked one), one masked block
CASES = [_sweep_case(200, skv, d) for d in (40, 64, 80) for skv in (256, 77, 50)]


def _trend_inputs(sign):
    def make(c, regime, Bn, seed):
        g = torch.Generator().manual_seed(seed)
        q = torch.randn(Bn, c.Sq, c.H, c.D, generator=g)
        k = torch.randn(Bn, c.Skv, c.H, c.D, generator=g)
        v = torch.randn(Bn, c.Skv, c.H, c.D, generator=g)
        scale = c.D ** -0.5
        # head coordinate 0 carries the trend: q[.., 0] = 4, so a key's logit moves by 4 * scale * k[.., 0]
        q[..., 1:] *= 0.25
        q[..., 0] = 4.0
        k[..., 0] = (sign * STEP / 64 * torch.arange(c.Skv, dtype=torch.float32) / (4.0 * scale))[None, :, None]
        q, k, v = q.to(BF), k.to(BF), v.to(BF)
        _check_trend(q, k, scale, sign)
        return q, k, v
    return make


def _check_trend(q, k, scale, sign):
    """Per row, each 64-key block's maximum against the maximum of the blocks before it."""
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) * scale
    nblk = (s.shape[-1] + 63) // 64
    run = s[..., :64].amax(-1)
    for j in range(1, nblk):
        m = s[..., 64 * j:64 * (j + 1)].amax(-1)
        if sign > 0:
            assert (m > run).all(), f"block {j} does not raise every row's maximum"
        else:
            assert (m < run).all(), f"block {j} reaches a row's maximum"
        run = torch.maximum(run, m)


@pytest.mark.parametrize("trend", ["rising", "falling"])
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_softmax_block_paths(cuda, case, trend, monkeypatch):
    monkeypatch.setattr(test_attn_gpu, "_logits_inputs", _trend_inputs(1.0 if trend == "rising" else -1.0))
    check_case(case, trend, cuda)
