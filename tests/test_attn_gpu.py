"""Flash attention forward and backward (pcm_attn_fwd / pcm_attn_bwd) against a float64 reference, at
the tensor layouts the UNet builds and at the shapes and logit regimes where an online softmax goes
wrong.

Reference: float64 attention on the bf16 inputs, computed one group of (batch, head) pairs at a time.
Error budget: a baseline doing the same math in torch with the kernels' roundings: bf16 inputs,
products on the tensor cores with fp32 accumulation, P rounded to bf16 before P.V, O rounded to bf16,
delta = rowsum(dO o O) summed in the delta kernel's order, P and dS rounded to bf16 before the
dV / dK / dQ products, outputs rounded to bf16.  For O, dQ, dK and dV, both the largest and the mean
absolute error against float64 must stay within twice the baseline's, plus 1e-6 of the reference's
largest magnitude and an fp32 floor; the lse within twice the baseline's largest error, the floor and
1e-6.  The floor covers what a bf16 budget cannot: where dS = P (dP - delta) cancels (a single key, or
one key far above the rest), dQ and dK are one fp32 rounding of dP - delta, and whether the baseline's
own rounding there comes out exact is luck, since the tensor cores and the delta kernel sum in
different orders.  It is 4 fp32 units of the cancelling terms, root-sum-squared into dQ / dK, and 4
units of the largest logit for the lse; away from cancellation it is far below the bf16 budget.

Every destination (out, dq, dk, dv, lse, delta) starts as NaN, with columns outside the head window,
one extra row and a tail of NaN: after the calls the window must be finite (every element written) and
everything else still NaN bit for bit (nothing written outside).  Input columns outside the q / k / v
windows are NaN as well, so a kernel reading outside its window fails the comparison.

The case table (CASES) is plain data; test_attn_layouts_cpu.py checks on CPU that it covers every
attention layout of the SD1.5 and SDXL training steps."""
import math
from typing import NamedTuple

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
LOG2E = 1.4426950408889634

# head sizes both directions support (pcm_attn_fwd / pcm_attn_bwd reject the others on the host)
SUPPORTED_HEAD_DIMS = tuple(list(range(8, 97, 8)) + [120, 128, 152, 160])

# N(0, 1) logits; logit std ~10; one key ~30 above the rest in the last (partial) key tile; two equal
# such keys, one in the first and one in the last tile; every logit ~ -20 (a zero-filled key past Skv
# that escaped the mask would dominate)
REGIMES = ("normal", "large", "late_spike", "two_spikes", "negative")


class Case(NamedTuple):
    B: int
    H: int
    Sq: int
    Skv: int
    D: int
    layout: str            # "dense" | "fused": q/k/v column views of [B*S, 3C + gutter] | "chunk"
    gutter: int = 0        # fused: columns past 3C
    W: int = 0             # chunk: k / v are windows of [B*Skv, W] (q and out dense) ...
    off: int = 0           # ... at column off (k) and off + C (v)
    merged: bool = False   # forward at 3B samples, backward on the leading B (row slices, lse[:B])


def layout_class(c):
    """(d, Sq, Skv, layout, chunk window position, merged): what test_attn_layouts_cpu.py matches."""
    pos = None
    if c.layout == "chunk":
        pos = "first" if c.off == 0 else "last" if c.off + 2 * c.H * c.D == c.W else "interior"
    return (c.D, c.Sq, c.Skv, c.layout, pos, c.merged)


def _fused(B, H, S, D, gutter=0, merged=False):
    return Case(B, H, S, S, D, "fused", gutter=gutter, merged=merged)


def _chunk(B, H, Sq, Skv, D, W, off, merged=False):
    return Case(B, H, Sq, Skv, D, "chunk", W=W, off=off, merged=merged)


# The UNet's layouts at B = 2 (the real batch changes no code path): self-attention on the fused qkv
# matrix (ld = 3C); cross-attention k / v in a context-chunk matrix whose width and window offsets are
# those of the SD1.5 / SDXL steps (first, interior and last window); forward on the merged 3B batch.
PROD_CASES = [
    # SD1.5: 8 heads; d = 40 / 80 / 160 at 64x64 / 32x32 / 16x16 / 8x8 latents
    _fused(2, 8, 4096, 40, merged=True),
    _fused(2, 8, 1024, 80, merged=True),
    _fused(2, 8, 256, 160, merged=True),
    _fused(2, 8, 64, 160, merged=True),
    _chunk(2, 8, 4096, 77, 40, 3200, 0, merged=True),
    _chunk(2, 8, 4096, 77, 40, 3200, 1280, merged=True),
    _chunk(2, 8, 4096, 77, 40, 3200, 2560, merged=True),
    _chunk(2, 8, 1024, 77, 80, 6400, 0, merged=True),
    _chunk(2, 8, 1024, 77, 80, 6400, 2560, merged=True),
    _chunk(2, 8, 1024, 77, 80, 6400, 5120, merged=True),
    _chunk(2, 8, 256, 77, 160, 15360, 0, merged=True),
    _chunk(2, 8, 256, 77, 160, 15360, 7680, merged=True),
    _chunk(2, 8, 256, 77, 160, 15360, 12800, merged=True),
    _chunk(2, 8, 64, 77, 160, 15360, 5120, merged=True),
    # SDXL: d = 64, 10 heads at 64x64 and 20 heads at 32x32
    _fused(2, 10, 4096, 64, merged=True),
    _fused(2, 20, 1024, 64, merged=True),
    _chunk(2, 10, 4096, 77, 64, 12800, 0, merged=True),
    _chunk(2, 10, 4096, 77, 64, 12800, 6400, merged=True),
    _chunk(2, 10, 4096, 77, 64, 12800, 11520, merged=True),
    _chunk(2, 20, 1024, 77, 64, 28160, 0, merged=True),
    _chunk(2, 20, 1024, 77, 64, 28160, 12800, merged=True),
    _chunk(2, 20, 1024, 77, 64, 28160, 25600, merged=True),
]

# Shape sweep at B = 2, H = 3 (not a power of two; the last head ends at the map's right edge): query
# and key counts around the 64-row tiles, 128-row CTAs and Skv below one tile.  Sq = Skv runs on the
# fused layout with 64 gutter columns, the rest on a context chunk (interior window); odd Sq also go
# through the merged batch.
_SQ = (1, 63, 64, 65, 127, 128, 129, 200)
_SKV = (1, 63, 64, 65, 77, 129)


def _sweep_case(Sq, Skv, D):
    C = 3 * D
    if Sq == Skv:
        return _fused(2, 3, Sq, D, gutter=64, merged=Sq % 2 == 1)
    return _chunk(2, 3, Sq, Skv, D, W=6 * C + 64, off=2 * C, merged=Sq % 2 == 1)


SWEEP_CASES = [_sweep_case(sq, skv, d) for d in (40, 64, 80, 160) for sq in _SQ for skv in _SKV] + \
    [_sweep_case(sq, skv, d) for d in (8, 72, 128) for sq in (1, 65, 129, 200) for skv in (1, 64, 77, 129)]

# the dense [B*S, H*D] cases of the first attention test
DENSE_CASES = [Case(*s, layout="dense") for s in [
    (2, 8, 256, 256, 40), (2, 8, 200, 77, 40), (1, 8, 1024, 1024, 80), (2, 8, 64, 64, 160),
    (2, 8, 64, 77, 160), (2, 2, 256, 256, 32), (1, 2, 128, 77, 64), (1, 8, 4096, 4096, 40)]]

CASES = PROD_CASES + SWEEP_CASES + DENSE_CASES


def _case_id(c):
    s = f"{c.layout}-B{c.B}H{c.H}-{c.Sq}x{c.Skv}-d{c.D}"
    if c.layout == "fused" and c.gutter:
        s += f"-g{c.gutter}"
    if c.layout == "chunk":
        s += f"-W{c.W}@{c.off}"
    return s + ("-merged" if c.merged else "")


# ---------------------------------------------------------------------------------------------
# inputs and destinations
# ---------------------------------------------------------------------------------------------
NAN_BF16 = torch.tensor(float("nan"), dtype=BF).view(torch.int16).item()
NAN_F32 = torch.tensor(float("nan"), dtype=torch.float32).view(torch.int32).item()


class Dest:
    """A NaN-filled destination matrix with one row more than used; `window` lists the column
    ranges the kernels must write in the used rows."""

    def __init__(self, rows, cols, dev, windows):
        self.buf = torch.full((rows + 1, cols), float("nan"), device=dev, dtype=BF)
        self.rows, self.windows = rows, windows

    def view(self, c0, c1):
        return self.buf[:self.rows, c0:c1]

    def check(self, what):
        mask = torch.zeros_like(self.buf, dtype=torch.bool)
        for c0, c1 in self.windows:
            mask[:self.rows, c0:c1] = True
        assert torch.isfinite(self.buf[mask]).all(), f"{what}: element of the window not written (NaN left)"
        outside = self.buf.view(torch.int16)[~mask]
        assert (outside == NAN_BF16).all(), f"{what}: {int((outside != NAN_BF16).sum())} elements written outside the window"


def _nan_f32(n, dev, tail=16):
    return torch.full((n + tail,), float("nan"), device=dev, dtype=torch.float32)


def _check_tail(buf, n, what):
    assert torch.isfinite(buf[:n]).all(), f"{what}: element not written"
    assert (buf[n:].view(torch.int32) == NAN_F32).all(), f"{what}: written past its end"


def _logits_inputs(c, regime, Bn, seed):
    """q [Bn, Sq, H, D], k / v [Bn, Skv, H, D] (fp32, bf16-representable) shaped for the regime."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(Bn, c.Sq, c.H, c.D, generator=g)
    k = torch.randn(Bn, c.Skv, c.H, c.D, generator=g)
    v = torch.randn(Bn, c.Skv, c.H, c.D, generator=g)
    scale = c.D ** -0.5
    if regime == "large":
        q *= 10.0
    elif regime != "normal":
        # head coordinate 0 carries the shift: q[.., 0] = 4, so a key's logit moves by 4 * scale * k[.., 0]
        q[..., 0] = 4.0
        k[..., 0] = 0.0
        peak = 30.0 / (4.0 * scale)
        if regime == "negative":
            k[..., 0] = -20.0 / (4.0 * scale)
        else:
            if regime == "two_spikes":
                k[:, 0] = k[:, -1]
                k[:, 0, :, 0] = peak
            k[:, -1, :, 0] = peak
    return q.to(BF), k.to(BF), v.to(BF)


def _setup(c, regime, dev, seed=0):
    """Kernel inputs and NaN destinations, laid out as the UNet lays them out."""
    B, H, Sq, Skv, D = c.B, c.H, c.Sq, c.Skv, c.D
    C, Bf = H * D, (3 * B if c.merged else B)
    q4, k4, v4 = _logits_inputs(c, regime, Bf, seed)
    g = torch.Generator().manual_seed(seed + 1)
    do = torch.randn(B * Sq, C, generator=g).to(BF).to(dev)
    nan = lambda r, w: torch.full((r, w), float("nan"), device=dev, dtype=BF)
    if c.layout == "fused":
        assert Sq == Skv
        ld = 3 * C + c.gutter
        m = nan(Bf * Sq, ld)
        q, k, v = m[:, :C], m[:, C:2 * C], m[:, 2 * C:3 * C]
        d = Dest(B * Sq, ld, dev, [(0, 3 * C)])
        dq, dk, dv = d.view(0, C), d.view(C, 2 * C), d.view(2 * C, 3 * C)
        dests = {"dq/dk/dv": d}
    elif c.layout == "chunk":
        q = nan(Bf * Sq, C)
        m = nan(Bf * Skv, c.W)
        k, v = m[:, c.off:c.off + C], m[:, c.off + C:c.off + 2 * C]
        dkv = Dest(B * Skv, c.W, dev, [(c.off, c.off + 2 * C)])
        dqd = Dest(B * Sq, C, dev, [(0, C)])
        dq, dk, dv = dqd.view(0, C), dkv.view(c.off, c.off + C), dkv.view(c.off + C, c.off + 2 * C)
        dests = {"dq": dqd, "dk/dv": dkv}
    else:
        q, k, v = nan(Bf * Sq, C), nan(Bf * Skv, C), nan(Bf * Skv, C)
        dqd, dkd, dvd = (Dest(B * s, C, dev, [(0, C)]) for s in (Sq, Skv, Skv))
        dq, dk, dv = dqd.view(0, C), dkd.view(0, C), dvd.view(0, C)
        dests = {"dq": dqd, "dk": dkd, "dv": dvd}
    q.copy_(q4.reshape(Bf * Sq, C))
    k.copy_(k4.reshape(Bf * Skv, C))
    v.copy_(v4.reshape(Bf * Skv, C))
    outd = Dest(Bf * Sq, C, dev, [(0, C)])
    lse_buf, delta_buf = _nan_f32(Bf * H * Sq, dev), _nan_f32(B * H * Sq, dev)
    return dict(q=q, k=k, v=v, do=do, out=outd.view(0, C), outd=outd, dq=dq, dk=dk, dv=dv, dests=dests,
                lse_buf=lse_buf, lse=lse_buf[:Bf * H * Sq].view(Bf, H, Sq), delta_buf=delta_buf,
                delta=delta_buf[:B * H * Sq].view(B, H, Sq), Bf=Bf)


def _run(c, X):
    from pcm_b200 import ops
    B, H, Sq, Skv, D = c.B, c.H, c.Sq, c.Skv, c.D
    scale = D ** -0.5
    ops.attn_fwd(X["q"], X["k"], X["v"], X["out"], X["lse"], X["Bf"], H, Sq, Skv, D, scale)
    ops.attn_bwd(X["q"][:B * Sq], X["k"][:B * Skv], X["v"][:B * Skv], X["out"][:B * Sq], X["do"], X["lse"][:B],
                 X["delta"], X["dq"], X["dk"], X["dv"], B, H, Sq, Skv, D, scale)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------
# float64 reference and the kernels' rounding baseline, on [N, S, D] head-major stacks
# ---------------------------------------------------------------------------------------------
def _heads(x, Bn, S, H, D):
    """[Bn*S, >=H*D] view -> [Bn*H, S, D]."""
    return x.reshape(Bn, S, H, D).permute(0, 2, 1, 3).reshape(Bn * H, S, D)


def _ref64(q, k, v, do, scale):
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.transpose(-1, -2) * scale
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    o = p @ v
    lse = (m + torch.log(l)).squeeze(-1) / math.log(2.0)
    # fp32 rounding floor (4 units of fp32 rounding): of the logits for the lse, and of the two terms
    # that cancel in dS = P (dP - delta), propagated to dQ / dK as a root sum of squares
    floor = dict(lse=2.0 ** -22 * s.abs().amax().item() / math.log(2.0))
    if do is None:
        return dict(o=o, lse=lse), floor
    do = do.double()
    dv = p.transpose(-1, -2) @ do
    dp, delta = do @ v.transpose(-1, -2), (do * o).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    t2 = (p * (dp.abs() + delta.abs())) ** 2
    floor["dq"] = 2.0 ** -22 * scale * (t2 @ k ** 2).sqrt().amax().item()
    floor["dk"] = 2.0 ** -22 * scale * (t2.transpose(-1, -2) @ q ** 2).sqrt().amax().item()
    return dict(o=o, lse=lse, dq=ds @ k * scale, dk=ds.transpose(-1, -2) @ q * scale, dv=dv), floor


def _mm(a, b):
    """bf16 x bf16 product accumulated in fp32 on the tensor cores, as the kernels' MMAs do."""
    return torch.bmm(a.to(BF), b.to(BF), out_dtype=torch.float32)


def _rowdot_fp32(o, do):
    """rowsum(dO o O) summed as attn_delta_kernel sums it: the bf16 products are exact in fp32, pairs
    are added, then accumulated left to right."""
    prod = o.float() * do.float()
    acc = torch.zeros(prod.shape[:-1], dtype=torch.float32, device=prod.device)
    for j in range(0, prod.shape[-1], 2):
        acc = acc + (prod[..., j] + prod[..., j + 1])
    return acc


def _baseline(q, k, v, do, scale):
    f32 = torch.float32
    c = torch.tensor(scale, dtype=f32) * torch.tensor(LOG2E, dtype=f32)
    s = _mm(q, k.transpose(-1, -2)) * c.to(q.device)
    m = s.amax(-1, keepdim=True)
    p = torch.exp2(s - m)
    l = p.sum(-1, keepdim=True)
    o = (_mm(p, v) / l).to(BF)
    lse = (m + torch.log2(l)).squeeze(-1)
    if do is None:
        return dict(o=o, lse=lse)
    p = torch.exp2(s - lse[..., None])
    ds = p * (_mm(do, v.transpose(-1, -2)) - _rowdot_fp32(o, do)[..., None])
    return dict(o=o, lse=lse, dq=(_mm(ds, k) * scale).to(BF), dk=(_mm(ds.transpose(-1, -2), q) * scale).to(BF),
                dv=_mm(p.transpose(-1, -2), do).to(BF))


class _Err:
    """max / sum |x - ref| and max |ref| accumulated over head groups."""

    def __init__(self):
        self.max = self.sum = self.ref = self.floor = 0.0
        self.n = 0

    def add(self, x, ref):
        e = (x.double() - ref).abs()
        self.max = max(self.max, e.max().item())
        self.sum += e.sum().item()
        self.n += e.numel()
        self.ref = max(self.ref, ref.abs().max().item())

    @property
    def mean(self):
        return self.sum / self.n


def _errors(c, X):
    """Errors of the kernels and of the baseline against float64, per output tensor."""
    B, H, Sq, Skv, D, Bf = c.B, c.H, c.Sq, c.Skv, c.D, X["Bf"]
    scale = D ** -0.5
    hq, hk, hv = (_heads(X[n], Bf, s, H, D) for n, s in (("q", Sq), ("k", Skv), ("v", Skv)))
    hdo = _heads(X["do"], B, Sq, H, D)
    kern = dict(o=_heads(X["out"], Bf, Sq, H, D), lse=X["lse"].reshape(Bf * H, Sq),
                dq=_heads(X["dq"], B, Sq, H, D), dk=_heads(X["dk"], B, Skv, H, D), dv=_heads(X["dv"], B, Skv, H, D))
    err = {n: (_Err(), _Err()) for n in kern}    # (kernel, baseline)
    nb = B * H                                    # backward heads: the leading B samples
    step = max(1, (1 << 24) // (Sq * Skv))
    for h0 in range(0, Bf * H, step):
        h1 = min(h0 + step, Bf * H)
        bwd = h0 < nb
        hb = min(h1, nb) if bwd else h1
        for sl, do in [(slice(h0, hb), hdo[h0:hb] if bwd else None)] + \
                ([(slice(hb, h1), None)] if hb < h1 else []):   # + forward-only heads of the group
            ref, floor = _ref64(hq[sl], hk[sl], hv[sl], do, scale)
            base = _baseline(hq[sl], hk[sl], hv[sl], do, scale)
            for n in ref:
                err[n][0].add(kern[n][sl], ref[n])
                err[n][1].add(base[n], ref[n])
                err[n][0].floor = max(err[n][0].floor, floor.get(n, 0.0))
    return err


def _ratios(err):
    """Kernel error over baseline error (max and mean) per tensor, for reports."""
    out = {}
    for n, (ke, be) in err.items():
        out[n] = (ke.max / be.max if be.max > 0 else (0.0 if ke.max == 0 else math.inf),
                  ke.mean / be.mean if be.mean > 0 else (0.0 if ke.mean == 0 else math.inf))
    return out


def check_case(c, regime, dev, seed=0):
    X = _setup(c, regime, dev, seed)
    _run(c, X)
    X["outd"].check("out")
    for name, d in X["dests"].items():
        d.check(name)
    Bf, H, Sq = X["Bf"], c.H, c.Sq
    _check_tail(X["lse_buf"], Bf * H * Sq, "lse")
    _check_tail(X["delta_buf"], c.B * H * Sq, "delta")
    # delta = rowsum(dO o O) of the kernel's own O: bf16 products are exact in fp32, so only the
    # D-term fp32 sum rounds
    o = _heads(X["out"][:c.B * Sq], c.B, Sq, H, c.D).double()
    prod = _heads(X["do"], c.B, Sq, H, c.D).double() * o
    dref = prod.sum(-1).view(c.B, H, Sq)
    bound = c.D * 2.0 ** -23 * prod.abs().sum(-1).view(c.B, H, Sq) + 1e-30
    assert ((X["delta"].double() - dref).abs() <= bound).all(), "delta != rowsum(dO o O)"
    err = _errors(c, X)
    for n, (ke, be) in err.items():
        if n == "lse":
            assert ke.max <= 2 * be.max + ke.floor + 1e-6, (n, ke.max, be.max, ke.floor)
            continue
        tol = 1e-6 * ke.ref + ke.floor
        assert ke.max <= 2 * be.max + tol, (n, "max", ke.max, be.max, _ratios(err))
        assert ke.mean <= 2 * be.mean + tol, (n, "mean", ke.mean, be.mean, _ratios(err))
    return err


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_attention_matches_float64(cuda, case, regime):
    check_case(case, regime, cuda)


@pytest.mark.parametrize("D", range(8, 161, 8))
def test_head_dim_support(cuda, D):
    """Each head size either runs forward and backward to parity, or both directions reject it on
    the host with the same message and write nothing."""
    from pcm_b200 import _lib, ops
    c = Case(1, 2, 65, 77, D, "chunk", W=6 * D + 64, off=2 * D)
    if D in SUPPORTED_HEAD_DIMS:
        check_case(c, "normal", cuda)
        return
    X = _setup(c, "normal", cuda)
    msgs = []
    for call in (lambda: ops.attn_fwd(X["q"], X["k"], X["v"], X["out"], X["lse"], 1, 2, 65, 77, D, 0.1),
                 lambda: ops.attn_bwd(X["q"], X["k"], X["v"], X["out"], X["do"], X["lse"], X["delta"], X["dq"],
                                      X["dk"], X["dv"], 1, 2, 65, 77, D, 0.1)):
        with pytest.raises(_lib.PcmError) as e:
            call()
        msgs.append(str(e.value).split("): ", 1)[1])
    torch.cuda.synchronize()
    assert msgs[0] == msgs[1] and f"head dim {D}" in msgs[0], msgs
    for t in [X["outd"].buf, *(d.buf for d in X["dests"].values())]:
        assert (t.view(torch.int16) == NAN_BF16).all()
    assert (X["lse_buf"].view(torch.int32) == NAN_F32).all() and (X["delta_buf"].view(torch.int32) == NAN_F32).all()


@pytest.mark.parametrize("case", [PROD_CASES[1], PROD_CASES[11], PROD_CASES[15], PROD_CASES[19],
                                  _sweep_case(129, 77, 40), _sweep_case(65, 65, 160)], ids=_case_id)
def test_attention_is_reproducible(cuda, case):
    """Forward plus backward twice on the same inputs: bitwise equal results (no atomics)."""
    runs = []
    for _ in range(2):
        X = _setup(case, "large", cuda)
        _run(case, X)
        runs.append([X["outd"].buf, *(d.buf for d in X["dests"].values()), X["lse_buf"], X["delta_buf"]])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int16) if a.dtype == BF else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == BF else b.view(torch.int32))
