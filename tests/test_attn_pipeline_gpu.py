"""Attention at the sizes where the pipelined wgmma kernels change phase: streamed sequences that wrap
the three-stage K / V (forward, dQ) and Q / dO (dK / dV) rings more than once, CTAs whose second consumer
warpgroup has no valid row, and head sizes on either side of the trimmed d <= 40 products.  Every case
must return and match float64 as tests/test_attn_gpu.py requires (same check, same NaN-guarded layouts)."""
import pytest

from test_attn_gpu import _case_id, _sweep_case, check_case

pytestmark = pytest.mark.gpu

# streamed lengths past one ring turn (3 stages = 192 rows): 193 wraps once, 450 wraps twice and ends
# ragged; the other side spans one CTA with an empty second warpgroup (1, 64), a one-row tail in the
# second warpgroup (65), and a second CTA (200)
WRAP = [(sq, skv) for sq in (1, 64, 65, 200) for skv in (193, 450)] + \
       [(sq, skv) for sq in (193, 450) for skv in (1, 65)]
CASES = [_sweep_case(sq, skv, d) for d in (8, 40, 48, 64) for sq, skv in WRAP] + \
        [_sweep_case(sq, skv, d) for d in (80, 128) for sq, skv in ((65, 193), (200, 450))]


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_attention_across_ring_wraps(cuda, case):
    check_case(case, "late_spike", cuda)
