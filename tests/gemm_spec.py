"""Pointer-free launch specs of `pcm_gemm` / `pcm_wgrad`, a float64 reference for them and an elementwise
error bound.  Test infrastructure: nothing under pcm_b200/ imports it.

A spec is plain data: the descriptor as tests/golden/make_launch_trace.py records it (every field,
pointers as [buffer label, byte offset]) with the labels renumbered per launch, plus `spans`, the bytes of
every buffer the launch's views cover.  Aliasing survives: the four parity planes of a stride-2 dgrad are
offsets into one buffer, grouped column views share theirs, an in-place residual has the label of `out`.
A launch with `dep_a_src1` carries `pre`, the launch issued immediately before it (the LoRA
down-projection that writes that A source); the two share one label space.

`materialise` turns a spec into poisoned buffers, `reference` computes the launch in float64 from the
descriptor semantics of include/pcm_b200.h, `check` compares elementwise, `guards` proves nothing outside
the destination window changed.  Everything runs on any torch device, so the oracle itself is tested on
the CPU (tests/test_gemm_specs_cpu.py)."""
import contextlib
import copy
import importlib.util
import json
import os

import torch

_GEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_launch_trace.py")
_s = importlib.util.spec_from_file_location("make_launch_trace", _GEN)
trace = importlib.util.module_from_spec(_s)
_s.loader.exec_module(trace)

BF16 = torch.bfloat16
POISON = 0x7FC0            # int16 pattern: a NaN as bf16, and 0x7FC07FC0 is a NaN as fp32 too
TAIL = 512                 # poisoned bytes after every buffer's span
NUM_SMS = 132              # the H100 SXM count the recorded plans were tiled for
_GEMM_PTRS = ("out", "bias", "rowvec", "residual", "splitk_ws")


# ---------------------------------------------------------------------------------------------
# spec_of / launch_class
# ---------------------------------------------------------------------------------------------
def _row_offsets(M, epiW, epiHW, osW, osH, osB):
    m = torch.arange(M, dtype=torch.int64)
    b, r = m // epiHW, m % epiHW
    return b * osB + (r // epiW) * osH + (r % epiW) * osW, b


def _asrc_elems(a, lin):
    if lin:
        return (a["W"] - 1) * a["sW"] + a["C"]
    return (a["B"] - 1) * a["sB"] + (a["H"] - 1) * a["sH"] + (a["W"] - 1) * a["sW"] + a["C"]


def _bsrc_elems(b):
    return b["K"] * b["N"] if b["kblocked"] else (b["N"] - 1) * b["ld"] + b["K"]


def wgrad_qw(d):
    return min(64, d["q"]["C"] - d["q_c0"])


def resolved_ksplit(d):
    """The K split `launch_gemm` runs: none without a workspace or with N- / M-ranged entries, no empty
    split.  (A spec's `splitk_ws` is never recorded: the dry run allocates none; `materialise` adds it.)"""
    nkb = sum(e["nchunks"] for e in d["prog"])
    if d["ksplit"] <= 1 or any(e["n_hi"] for e in d["prog"]):
        return 1
    ks = min(d["ksplit"], nkb)
    per = -(-nkb // ks)
    return -(-nkb // per)


def _views(op, d):
    """(pointer, byte length) of every view of one launch; pointers are [label, offset] or None."""
    if op == "wgrad":
        hi = max(d["tap_off"]) + (d["p"]["C"] - 1) * d["os_row"] + (wgrad_qw(d) - 1) * d["os_col"] + 1
        return [(d["p"]["ptr"], 2 * _asrc_elems(d["p"], d["lin"])), (d["q"]["ptr"], 2 * _asrc_elems(d["q"], d["lin"])),
                (d["out"], 4 * hi)]
    off, b = _row_offsets(d["M"], d["epiW"], d["epiHW"], d["osW"], d["osH"], d["osB"])
    hi = int(off.max()) + d["N"]
    v = [(a["ptr"], 2 * _asrc_elems(a, d["lin"])) for a in d["a"]]
    v += [(bs["ptr"], 2 * _bsrc_elems(bs)) for bs in d["b"]]
    v += [(d["out"], (4 if d["out_fp32"] else 2) * hi), (d["bias"], 4 * d["N"]), (d["residual"], 2 * hi),
          (d["rowvec"], 2 * (int(b.max()) * d["rowvec_ld"] + d["N"]))]
    return v


def _pointers(op, d):
    """The mutable [label, offset] lists of a descriptor, in a fixed order."""
    if op == "wgrad":
        return [p for p in (d["p"]["ptr"], d["q"]["ptr"], d["out"]) if p]
    ps = [a["ptr"] for a in d["a"]] + [b["ptr"] for b in d["b"]] + [d[k] for k in _GEMM_PTRS]
    return [p for p in ps if p]


def spec_of(rec, prev=None):
    """One recorded launch (`rec`, a trace record with op / desc) as a spec; `prev` is the record issued
    immediately before it, required exactly when the launch has dep_a_src1."""
    op, d = rec["op"], copy.deepcopy(rec["desc"])
    assert op in ("gemm", "wgrad")
    dep = op == "gemm" and d["dep_a_src1"] != 0
    assert dep == (prev is not None), "a dep_a_src1 launch is recorded with its producer, and only such a launch"
    spec = dict(op=op, desc=d)
    launches = [(op, d)]
    if dep:
        assert prev["op"] == "gemm" and prev["desc"]["out"][0] == d["a"][d["dep_a_src1"] - 1]["ptr"][0]
        spec["pre"] = copy.deepcopy(prev["desc"])
        launches.append(("gemm", spec["pre"]))
    if op == "gemm":
        d["splitk_ws"] = None
    labels, spans = {}, {}
    for o, dd in launches:
        for p in _pointers(o, dd):
            p[0] = labels.setdefault(p[0], len(labels))
        for p, n in _views(o, dd):
            if p:
                spans[p[0]] = max(spans.get(p[0], 0), p[1] + n)
    spec["spans"] = [spans[i] for i in range(len(labels))]
    return spec


def _class_of(op, d):
    d = copy.deepcopy(d)
    for p in _pointers(op, d):
        del p[1:]                       # which buffer (aliasing), not where in it
    d["alpha"] = d["alpha"] != 1.0
    if op == "gemm":
        d["ksplit"] = resolved_ksplit(d)
        # what launch_gemm derives and the kernel branches on
        d["narrow"] = any(min(d["a"][e["a_src"]]["C"] - e["a_c0"], d["b"][e["b_src"]]["K"] - e["b_k0"]) < 64 * e["nchunks"]
                          for e in d["prog"])
        d["m_hi"] = [_m_hi(d, e) for e in d["prog"]]
    else:
        d["qw"] = wgrad_qw(d)
    return d


def _m_hi(d, e):
    a = d["a"][e["a_src"]]
    rows = a["W"] if d["lin"] else a["B"] * d["geoW"] * d["geoH"]
    return rows if (rows < d["M"] and rows % 128 == 0 and d["ksplit"] <= 1) else 0


def launch_class(spec):
    """The key launches are de-duplicated by: every descriptor field that selects code in launch_gemm, the
    kernels or the epilogue (dims, strides, tiling, the whole K program, the epilogue options), the
    aliasing pattern of the buffers, `alpha != 1` instead of its value, and the derived NARROW / m_hi /
    resolved ksplit.  Only the byte offsets of the pointers inside their buffers are dropped: two launches
    that differ in nothing else run the same instructions on another window."""
    key = dict(op=spec["op"], desc=_class_of(spec["op"], spec["desc"]))
    if "pre" in spec:
        key["pre"] = _class_of("gemm", spec["pre"])
    return json.dumps(key, sort_keys=True, separators=(",", ":"))


def distinct_specs(records):
    """The first spec of every launch class of a recorded trace, in launch order.  A launch's predecessor is
    the previous record on its own stream (`side`: the weight-gradient stream runs beside the main one)."""
    seen, out, last = set(), [], {}
    for r in records:
        prev = last.get(r["side"])
        if r["op"] in ("gemm", "wgrad"):
            s = spec_of(r, prev if (r["op"] == "gemm" and r["desc"]["dep_a_src1"]) else None)
            k = launch_class(s)
            if k not in seen:
                seen.add(k)
                out.append(s)
        if "side" in r and not r["op"].startswith("reducer."):
            last[r["side"]] = r
    return out


def family(spec):
    """Coarse name of a launch for the margin report."""
    d = spec["desc"]
    if spec["op"] == "wgrad":
        return "wgrad " + ("linear" if d["lin"] else f"{d['num_taps']}-tap")
    kind = "linear" if d["lin"] else ("conv %d-entry" % len(d["prog"]))
    extra = [n for n, on in (("pdl", "pre" in spec), ("splitk", resolved_ksplit(d) > 1), ("narrow", _class_of("gemm", d)["narrow"]),
                             ("n-ranged", any(e["n_hi"] for e in d["prog"])), ("fp32", d["out_fp32"]),
                             ("strided", not d["lin"] and d["osH"] != d["osW"] * d["epiW"])) if on]
    return " ".join([kind] + extra)


@contextlib.contextmanager
def recording():
    """Record ops.gemm / ops.wgrad calls made on CPU tensors (nothing launches): yields the Recorder; its
    `trace` holds the launch records `spec_of` takes."""
    import pytest
    rec = trace.Recorder()
    with pytest.MonkeyPatch.context() as mp:
        trace._install(mp, rec)
        yield rec


# ---------------------------------------------------------------------------------------------
# materialise
# ---------------------------------------------------------------------------------------------
class Tensors:
    """The buffers of a materialised spec.  `bufs[label]` is an int16 tensor (span + TAIL)."""

    def __init__(self, spec, device):
        self.device = device
        self.bufs = [torch.full(((n + 15) // 16 * 8 + TAIL // 2,), POISON, dtype=torch.int16, device=device)
                     for n in spec["spans"]]
        self.ws = self.ws_pre = self.sem = None

    def flat(self, ptr, dtype):
        """1-D typed view of a buffer from a pointer's byte offset to the buffer's end."""
        b = self.bufs[ptr[0]].view(torch.uint8)[ptr[1]:]
        return b[:b.numel() // 4 * 4].view(dtype)

    def addr(self, ptr):
        return 0 if ptr is None else self.bufs[ptr[0]].data_ptr() + ptr[1]

    def asrc(self, a, lin):
        f = self.flat(a["ptr"], BF16)
        if lin:
            return f.as_strided((1, 1, a["W"], a["C"]), (0, 0, a["sW"], 1))
        return f.as_strided((a["B"], a["H"], a["W"], a["C"]), (a["sB"], a["sH"], a["sW"], 1))

    def bsrc_view(self, b):
        """Writable view of the weights: [N, K], or [N, K/64, 64] of K-blocked storage."""
        f = self.flat(b["ptr"], BF16)
        if b["kblocked"]:
            return f[:b["K"] * b["N"]].view(b["K"] // 64, b["N"], 64).permute(1, 0, 2)
        return f.as_strided((b["N"], b["K"]), (b["ld"], 1))

    def bsrc(self, b):
        """The weights as an [N, K] matrix, whichever way they are stored (a copy when K-blocked)."""
        return self.bsrc_view(b).reshape(b["N"], b["K"])

    def out_index(self, d):
        """[M, N] element indices of the destination window into flat(d['out'], its dtype)."""
        off, _ = _row_offsets(d["M"], d["epiW"], d["epiHW"], d["osW"], d["osH"], d["osB"])
        return (off[:, None] + torch.arange(d["N"])[None]).to(self.device)

    def wgrad_index(self, d):
        """[taps, Cp, qw] element indices of a weight gradient's destination."""
        t = torch.tensor(d["tap_off"])[:, None, None]
        return (t + torch.arange(d["p"]["C"])[None, :, None] * d["os_row"]
                + torch.arange(wgrad_qw(d))[None, None, :] * d["os_col"]).to(self.device)


def _randn(shape, gen):
    return torch.randn(tuple(shape), generator=gen, device=gen.device)


def _fill(view, gen, scale=1.0):
    view.copy_((_randn(view.shape, gen) * scale).to(BF16))


def materialise(spec, device, seed=0):
    """Every buffer at its span plus a tail, all of it the NaN pattern; then seeded values only inside the
    declared dims of each operand (TMA may legally touch anything inside them), so row gutters, columns
    beside a window, rows past the last and the tail stay poisoned.  bias / rowvec / residual are real;
    `out` stays NaN unless it aliases the residual; the split-K workspace is NaN; a weight gradient's
    destination holds values of the result's scale, because the kernel accumulates into it.  In a pair,
    the intermediate the first launch writes stays NaN until that launch runs."""
    T = Tensors(spec, device)
    g = torch.Generator(device=device).manual_seed(seed)
    d = spec["desc"]
    if spec["op"] == "wgrad":
        _fill(T.asrc(d["p"], d["lin"]), g)
        _fill(T.asrc(d["q"], d["lin"]), g)
        idx = T.wgrad_index(d)
        T.flat(d["out"], torch.float32)[idx] = _randn(idx.shape, g) * abs(d["alpha"]) * d["M"] ** 0.5
        T.sem = torch.zeros(4096, dtype=torch.int32, device=device)
        return T
    launches = [d] + ([spec["pre"]] if "pre" in spec else [])
    for dd in launches:
        for a in dd["a"]:
            _fill(T.asrc(a, dd["lin"]), g)
        for b in dd["b"]:
            _fill(T.bsrc_view(b), g, b["K"] ** -0.5)
        if dd["bias"]:
            T.flat(dd["bias"], torch.float32)[:dd["N"]] = _randn((dd["N"],), g)
    for dd in reversed(launches):         # the producer's destination first: the consumer's may not alias it
        idx = T.out_index(dd)
        if dd["rowvec"]:
            nb = (dd["M"] - 1) // dd["epiHW"] + 1
            _fill(T.flat(dd["rowvec"], BF16).as_strided((nb, dd["N"]), (dd["rowvec_ld"], 1)), g)
        if dd["residual"]:
            T.flat(dd["residual"], BF16)[idx] = _randn(idx.shape, g).to(BF16)
        if not (dd["residual"] and dd["residual"] == dd["out"]):
            T.flat(dd["out"], torch.float32 if dd["out_fp32"] else BF16)[idx] = float("nan")
    T.ws = _workspace(d, device)
    if "pre" in spec:
        T.ws_pre = _workspace(spec["pre"], device)
    return T


def _workspace(d, device):
    # the header's size for the split asked for; a program too short to split still has to bring one
    ks = d["ksplit"]
    if ks <= 1 or any(e["n_hi"] for e in d["prog"]):
        return None
    return torch.full((ks * d["M"] * d["N"] + TAIL // 4,), float("nan"), dtype=torch.float32, device=device)


# ---------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------
def _rows(T, a, lin, geo, m, dw, dh, c0, kk):
    """[len(m), kk] bf16: row m of the implicit A matrix = channels c0.. of source pixel
    (b, h + dh, w + dw), zero outside the source's W / H / B (what the TMA box load delivers)."""
    if lin:
        b = h = torch.zeros_like(m)
        w = m
        H, B, sH, sB = 1, 1, 0, 0
    else:
        W, Hh = geo
        b, r = m // (W * Hh), m % (W * Hh)
        h, w = r // W + dh, r % W + dw
        H, B, sH, sB = a["H"], a["B"], a["sH"], a["sB"]
    valid = (w >= 0) & (w < a["W"]) & (h >= 0) & (h < H) & (b < B)
    idx = b * sB + h * sH + w * a["sW"]
    idx = torch.where(valid, idx, torch.zeros_like(idx))
    x = T.flat(a["ptr"], BF16)[idx[:, None] + (c0 + torch.arange(kk, device=m.device))[None]]
    return torch.where(valid[:, None], x, torch.zeros_like(x))


def _silu(x):
    return x * torch.sigmoid(x)


def reference(spec, T, desc=None, row_block=16384, rows=None):
    """(ref, S, base) of one pcm_gemm launch, each [M, N]: the float64 result, the same sum over absolute
    values (alpha |A| |B|^T + |bias| + |rowvec| + |residual|), and a torch baseline with the kernel's
    roundings (bf16 operands, fp32 accumulate, fp32 epilogue) before its one output rounding.
    Written from include/pcm_b200.h: entry e multiplies min(64 nchunks, a.C - a_c0, b.K - b_k0) K columns
    of source pixel (b, h + dh, w + dw), zero outside the source, against rows [n_lo, n_hi) of b.
    rows = (m0, m1): only output rows m0 .. m1 - 1 ([m1 - m0, N] results), for launches too large to hold
    in float64 at once."""
    d = desc or spec["desc"]
    dev = T.device
    M, N = d["M"], d["N"]
    m0, m1 = rows or (0, M)
    ref = torch.empty(m1 - m0, N, dtype=torch.float64, device=dev)
    S, base = torch.empty_like(ref), torch.empty(m1 - m0, N, dtype=torch.float32, device=dev)
    off, bimg = _row_offsets(M, d["epiW"], d["epiHW"], d["osW"], d["osH"], d["osB"])
    off, bimg = off.to(dev), bimg.to(dev)
    al = float(d["alpha"])
    for r0 in range(m0, m1, row_block):
        m = torch.arange(r0, min(m1, r0 + row_block), device=dev)
        acc = torch.zeros(len(m), N, dtype=torch.float64, device=dev)
        ab, a32 = torch.zeros_like(acc), torch.zeros(len(m), N, dtype=torch.float32, device=dev)
        for e in d["prog"]:
            a, b = d["a"][e["a_src"]], d["b"][e["b_src"]]
            kk = min(64 * e["nchunks"], a["C"] - e["a_c0"], b["K"] - e["b_k0"])
            lo, hi = (e["n_lo"], min(e["n_hi"], N)) if e["n_hi"] else (0, N)
            hi = min(hi, b["N"])         # columns past the weights' rows are TMA zero fill
            if kk <= 0 or hi <= lo:
                continue
            A = _rows(T, a, d["lin"], (d["geoW"], d["geoH"]), m, e["dw"], e["dh"], e["a_c0"], kk)
            Bm = T.bsrc(b)[lo:hi, e["b_k0"]:e["b_k0"] + kk]
            Ad, Bd = A.double(), Bm.double()
            acc[:, lo:hi] += Ad @ Bd.t()
            ab[:, lo:hi] += Ad.abs() @ Bd.abs().t()
            a32[:, lo:hi] += A.float() @ Bm.float().t()
        acc, ab, a32 = acc * al, ab * abs(al), a32 * d["alpha"]
        if d["bias"]:
            bias = T.flat(d["bias"], torch.float32)[:N]
            acc, ab, a32 = acc + bias.double(), ab + bias.double().abs(), a32 + bias
        if d["rowvec"]:
            rv = T.flat(d["rowvec"], BF16)[(bimg[m] * d["rowvec_ld"])[:, None] + torch.arange(N, device=dev)[None]]
            acc, ab, a32 = acc + rv.double(), ab + rv.double().abs(), a32 + rv.float()
        if d["residual"]:
            rs = T.flat(d["residual"], BF16)[off[m][:, None] + torch.arange(N, device=dev)[None]]
            acc, ab, a32 = acc + rs.double(), ab + rs.double().abs(), a32 + rs.float()
        if d["act"] == 1:
            acc, a32 = _silu(acc), _silu(a32)
        else:
            assert d["act"] == 0
        ref[m - m0], S[m - m0], base[m - m0] = acc, ab, a32
    return ref, S, base


def reference_wgrad(spec, T, desc=None):
    """(ref, S, base) [taps, Cp, qw] of one pcm_wgrad launch: out0 + alpha sum_m P[m(+tap), ch] Q[m, q_c0 + r]."""
    d = desc or spec["desc"]
    dev = T.device
    m = torch.arange(d["M"], device=dev)
    qw = wgrad_qw(d)
    Q = _rows(T, d["q"], d["lin"], (d["geoW"], d["geoH"]), m, 0, 0, d["q_c0"], qw)
    out0 = T.flat(d["out"], torch.float32)[T.wgrad_index(d)]
    ref, S, base = [], [], []
    for t in range(d["num_taps"]):
        P = _rows(T, d["p"], d["lin"], (d["geoW"], d["geoH"]), m, d["dw"][t], d["dh"][t], 0, d["p"]["C"])
        ref.append(float(d["alpha"]) * (P.double().t() @ Q.double()))
        S.append(abs(float(d["alpha"])) * (P.double().abs().t() @ Q.double().abs()))
        base.append(d["alpha"] * (P.float().t() @ Q.float()))
    ref, S, base = torch.stack(ref), torch.stack(S), torch.stack(base)
    return ref + out0.double(), S + out0.double().abs(), base + out0


# ---------------------------------------------------------------------------------------------
# check
# ---------------------------------------------------------------------------------------------
U_BF16 = 2.0 ** -8         # round to nearest at 8 significand bits: half an ulp of 2^-7
U_STEP = 2.0 ** -22        # per k16 step of the fp32 accumulator


def num_sms():
    """SMs of the device the launch runs on; the 132 of an H100 SXM where there is none (CPU tests)."""
    if torch.cuda.is_available():
        from pcm_b200 import ops
        return ops.num_sms()
    return NUM_SMS


def k_steps(spec, desc=None):
    """(k16 steps one accumulator sums, partial sums added afterwards) of a launch.  For a weight gradient with
    ksplit = 0 the split count is the one pcm_wgrad documents: about two waves of CTAs on the device's SMs,
    at least four 128-token blocks each."""
    d = desc or spec["desc"]
    if spec["op"] == "wgrad":
        nkb = -(-d["M"] // 128)
        tiles = -(-d["p"]["C"] // 128) * d["num_taps"]
        ks = d["ksplit"] if d["ksplit"] > 0 else max(1, min(-(-nkb // 4), -(-2 * num_sms() // tiles)))
        ks = min(ks, nkb)
        return 8 * -(-nkb // ks), ks
    ks = resolved_ksplit(d)
    return 4 * -(-sum(e["nchunks"] for e in d["prog"]) // ks), ks


def bound(ref, S, spec, desc=None):
    """Elementwise bound on |out - ref|.

    The operands are bf16, so every product is exact in fp32 and S = sum |a||b| (+ |epilogue terms|) bounds
    every partial sum.  A wgmma k16 step adds 16 exact products into the fp32 accumulator; the tensor core
    aligns and truncates the addends, which costs at most 2 ulp = 2^-22 of the running magnitude per step
    (twice the 2^-23 of one truncated fp32 add: one for the products' alignment, one for the accumulate).
    An accumulator sums `steps` of them; split-K (or the token splits of a weight gradient) then adds
    `parts` partial sums, one rounding each; alpha, bias, row vector and residual are four more fp32
    roundings.  So the value before the output rounding is within
        e = (steps + parts + 4) * 2^-22 * S
    of the exact one.  SiLU has slope <= 1.1 and the fast exponential adds a relative 2^-20.  A bf16
    result (or round_bf16) is then rounded to nearest once: 2^-8 of (|ref| + e).  Nothing scales with
    max|ref|: an element with a small S has a small bound.

    It is a worst-case bound, linear in the number of steps, while real errors grow like its square root.
    For a short K the output rounding dominates and the test resolves single bf16 ulps; for the longest
    programs (skip-concat 3x3 convolutions, about 1400 steps) e is several times the output rounding, so
    an error confined to a few elements and smaller than e passes here and is left to the mean test of
    `check`.  The GPU tests print each family's margin with its longest sum for that reason."""
    d = desc or spec["desc"]
    steps, parts = k_steps(spec, d)
    e = (steps + parts + 4) * U_STEP * S
    if spec["op"] == "gemm":
        if d["act"] == 1:
            e = 1.1 * e + 2.0 ** -20 * ref.abs()
        if not d["out_fp32"] or d["round_bf16"]:
            e = e + U_BF16 * (ref.abs() + e)
    return e + 1e-30


def check(out, ref, S, spec, base=None, desc=None):
    """Assert `out` (the destination window, any float dtype) is finite and within `bound` of `ref`
    elementwise, and, given the torch baseline, that its mean absolute error is at most twice the
    baseline's after the same output rounding (or a tenth of the mean bound, whichever is larger).
    Returns the largest err / bound."""
    d = desc or spec["desc"]
    out = out.double()
    assert torch.isfinite(out).all(), f"{int((~torch.isfinite(out)).sum())} non-finite destination elements"
    err, bnd = (out - ref).abs(), bound(ref, S, spec, d)
    ratio = err / bnd
    worst = float(ratio.max())
    if worst > 1.0:
        i = [int(x) for x in torch.unravel_index(ratio.argmax(), ratio.shape)]
        bad = (ratio > 1.0).nonzero()
        raise AssertionError(f"{int((ratio > 1).sum())} elements outside the bound, worst at {i}: out {float(out[tuple(i)])!r} "
                             f"ref {float(ref[tuple(i)])!r} bound {float(bnd[tuple(i)]):.3e} (x{worst:.1f}); "
                             f"index range {bad.min(0).values.tolist()}..{bad.max(0).values.tolist()}")
    if base is not None:
        if spec["op"] == "gemm" and (not d["out_fp32"] or d["round_bf16"]):
            base = base.to(BF16)
        mean, mean_base = float(err.mean()), float((base.double() - ref).abs().mean())
        if spec["op"] == "wgrad":
            # the baseline adds one finished sum to the destination; the kernel adds one partial sum per token
            # split, each add rounding at the destination's magnitude (an ulp of it, 2^-23, per split)
            mean_base += k_steps(spec, d)[1] * 2.0 ** -23 * float(ref.abs().mean())
        # (the tensor core's fp32 accumulator truncates, a bias a round-to-nearest baseline does not have: where
        # no output rounding hides it - weight gradients, unrounded fp32 results - a tenth of the mean bound applies)
        mean_base = max(mean_base, 0.05 * float(bnd.mean()))
        assert mean <= 2.0 * mean_base + 1e-30, f"mean |err| {mean:.3e} is more than twice the torch baseline's {mean_base:.3e}"
    return worst


# ---------------------------------------------------------------------------------------------
# launching (GPU tests) and guards
# ---------------------------------------------------------------------------------------------
def _fill_struct(s, d, T):
    import ctypes
    for name, typ in s._fields_:
        if name not in d:
            continue
        v = d[name]
        if typ is ctypes.c_void_p:
            setattr(s, name, T.addr(v))
        elif isinstance(v, dict):
            _fill_struct(getattr(s, name), v, T)
        elif isinstance(v, list):
            arr = getattr(s, name)
            for i, x in enumerate(v):
                if isinstance(x, dict):
                    _fill_struct(arr[i], x, T)
                else:
                    arr[i] = x
        else:
            setattr(s, name, v)
    return s


def gemm_desc(d, T, ws=None, **over):
    """ctypes pcm_gemm_desc of a spec's descriptor on materialised buffers, exactly as recorded; the
    split-K workspace is `ws` (default T.ws)."""
    from pcm_b200 import _lib
    s = _fill_struct(_lib.GemmDesc(), d, T)
    ws = T.ws if ws is None else ws
    if ws is not None:
        s.splitk_ws = ws.data_ptr()
    for k, v in over.items():
        setattr(s, k, v)
    return s


def wgrad_desc(d, T, sem=False):
    from pcm_b200 import _lib
    s = _fill_struct(_lib.WgradDesc(), d, T)
    s.sem = T.sem.data_ptr() if sem else 0
    return s


def launch(spec, T, stream=None, sem=False):
    """Run the spec's launch (after its producer, back to back, for a pair) through the C ABI."""
    import ctypes
    from pcm_b200 import _lib
    lib = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream if stream is None else stream)
    if spec["op"] == "wgrad":
        dd = wgrad_desc(spec["desc"], T, sem)
        _lib.check(lib.pcm_wgrad(ctypes.byref(dd), st), "pcm_wgrad")
        return
    if "pre" in spec:
        dp = gemm_desc(spec["pre"], T, ws=T.ws_pre)
        _lib.check(lib.pcm_gemm(ctypes.byref(dp), st), "pcm_gemm")
    dd = gemm_desc(spec["desc"], T)
    _lib.check(lib.pcm_gemm(ctypes.byref(dd), st), "pcm_gemm")


def snapshot(T):
    return [b.clone() for b in T.bufs]


def window(spec, T):
    """(flat typed view, element indices) of the destination window of the spec's launch."""
    d = spec["desc"]
    if spec["op"] == "wgrad":
        return T.flat(d["out"], torch.float32), T.wgrad_index(d)
    return T.flat(d["out"], torch.float32 if d["out_fp32"] else BF16), T.out_index(d)


def guards(spec, T, before):
    """Outside the destination windows (this launch's and, in a pair, its producer's) every byte of every
    buffer is what it was before the launch: operands unchanged, and the poison in columns past N, rows
    past M, gutters of a strided output, other parity planes and the tail still there bit for bit."""
    masks = [torch.zeros_like(b, dtype=torch.bool) for b in T.bufs]
    wins = [(spec["op"], spec["desc"])] + ([("gemm", spec["pre"])] if "pre" in spec else [])
    for op, d in wins:
        if op == "wgrad":
            es, idx = 4, T.wgrad_index(d)
        else:
            es, idx = (4 if d["out_fp32"] else 2), T.out_index(d)
        assert d["out"][1] % es == 0
        i16 = idx.reshape(-1) * (es // 2) + d["out"][1] // 2
        masks[d["out"][0]][i16] = True
        if es == 4:
            masks[d["out"][0]][i16 + 1] = True
    for lab, (b, b0, mk) in enumerate(zip(T.bufs, before, masks)):
        changed = (b != b0) & ~mk
        if changed.any():
            at = changed.nonzero().flatten()
            raise AssertionError(f"buffer {lab}: {len(at)} 2-byte words outside the destination window changed, "
                                 f"byte offsets {2 * int(at[0])}..{2 * int(at[-1])} (span {spec['spans'][lab]})")
