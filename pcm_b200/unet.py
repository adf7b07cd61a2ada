"""H100 (sm_90a) SD1.5 UNet (student / target with fused LoRA, frozen teacher) -- host orchestration.

Python only sequences C-ABI kernel launches (pcm_b200.ops); every FLOP runs in libpcm_b200.so.
Mirrors the call `unet(sample, timestep, encoder_hidden_states=...).sample` of diffusers'
UNet2DConditionModel wrapped by peft (train_pcm_lora_sd15.py:1192-1198 student, :1219-1244
teacher, :1263-1268 target) and its autograd backward (:1296), with:
  * activations NHWC bf16, one rounding per materialised tensor (bf16 autocast semantics);
  * LoRA unmerged (rank 8 <= r <= 256, r % 8 == 0): T = A(x) as an r-wide GEMM, then s*B*T enters the
    base GEMM as ceil(r/64) extra K blocks, the last one r % 64 wide (same wgmma accumulator), so
    `base(x) + B(A(x)) * scaling` is one kernel;
  * skip concats never materialised (two K segments / two GroupNorm sources);
  * backward = explicit tape: dgrad through every layer, wgrad for LoRA factors only.
Parameters use diffusers state-dict names; LoRA factors live in ONE flat fp32 buffer
(`lora_master`), their gradients in `lora_grad`.
"""
import copy
import types
import weakref
from collections import namedtuple
from dataclasses import dataclass, field
from typing import Optional

import torch

from . import ops
from .config import UNetConfig, check_lora_rank, is_lora_target, layer_table

BF16 = torch.bfloat16
TAPS3 = ops.TAPS3
# stride-2 3x3 pad-1: kernel index -> (input parity, shift in the parity plane)
_S2 = ((1, -1), (0, 0), (1, 0))
# per input parity p: the kernel indices that read parity plane p, with their shifts in that plane
_S2_PLANE = [[(k, sh) for k, (par, sh) in enumerate(_S2) if par == p] for p in range(2)]


def conv_prog(xs, k, stride, cin_total, s2=_S2):
    """(a_srcs, prog) of a k x k convolution over channel-concatenated NHWC sources xs.  A stride-2 3x3
    convolution reads the four parity planes of xs[0]; s2 maps its kernel index to (input parity, shift in
    the parity plane): the default is pad 1 (the UNet's downsamplers)."""
    if stride == 2:
        x = xs[0]
        planes = [x[:, p::2, q::2, :] for p in range(2) for q in range(2)]
        srcs = [ops.asrc_nhwc(pl) for pl in planes]
        prog = []
        for kh in range(3):
            for kw in range(3):
                p, dh = s2[kh]
                q, dw = s2[kw]
                prog.append((p * 2 + q, 0, dw, dh, cin_total // 64, 0, (kh * 3 + kw) * cin_total))
        return srcs, prog
    srcs = [ops.asrc_nhwc(x) for x in xs]
    taps = TAPS3 if k == 3 else [(0, 0)]
    prog, coff = [], 0
    for si, x in enumerate(xs):
        ci = x.shape[-1]
        for t, (dw, dh) in enumerate(taps):
            prog.append((si, 0, dw, dh, ci // 64, 0, t * cin_total + coff))
        coff += ci
    return srcs, prog


# tape records: what the backward of one op needs (views of the LoRA samples' rows only).  `op` names the
# op kind; T is the layer's LoRA down-projection x A^T (None: no adapter).
LinearRec = namedtuple("LinearRec", "op name xs T")
TembRec = namedtuple("TembRec", "op name xs T t_c0")     # time_emb_proj: its block of T starts at column t_c0
GroupRec = namedtuple("GroupRec", "op lead x T")         # lead: key of UNetB200.groups
ConvRec = namedtuple("ConvRec", "op name xs T stride")
GNRec = namedtuple("GNRec", "op name xs stats eps silu B HW")
LNRec = namedtuple("LNRec", "op name x stats")
AttnRec = namedtuple("AttnRec", "op q k v out lse B Sq Skv heads")
GegluRec = namedtuple("GegluRec", "op u")
# one BasicTransformerBlock
TBlockRec = namedtuple("TBlockRec", "norm1 attn1_qkv attn1 attn1_out norm2 attn2_q attn2_kv attn2 attn2_out "
                                    "norm3 ff_in geglu ff_out")


def _last(records):
    """The record a primitive just appended to `records` (None when the pass keeps no tape)."""
    return records[-1] if records is not None else None


class _Block:
    takes_skip = False      # the input was [hidden state, skip]: an up-path resnet
    pushes_skip = False     # the output went onto the skip list: end of a down-path group, downsampler


@dataclass
class ResnetRec(_Block):
    name: str
    norm1: GNRec
    temb: TembRec
    conv1: ConvRec
    norm2: GNRec
    shortcut: Optional[LinearRec]
    conv2: ConvRec
    takes_skip: bool


@dataclass
class TransformerRec(_Block):
    name: str
    norm: GNRec
    proj_in: LinearRec
    blocks: list            # TBlockRec per transformer block
    proj_out: LinearRec


@dataclass
class ResampleRec(_Block):
    name: str
    conv: ConvRec           # stride 2 (down), or after the nearest-2x upsample (up)
    up: bool


@dataclass
class CheckpointRec(_Block):
    """A block of a gradient-checkpointed forward: what rebuilding its full record in backward() takes."""
    kind: str               # "resnet" | "transformer" | "resample" (the UNetB200 method that runs it)
    name: str
    xs: list                # its inputs, student rows only, each an owned copy (an upsampler: before the 2x)
    takes_skip: bool
    up: bool = False


class _Lora:
    __slots__ = ("a_off", "b_off", "a_fwd", "sb_fwd", "sb_t", "a_t", "gA", "gB", "opnd_off",
                 "o_a_fwd", "o_sb_fwd", "o_sb_t", "o_a_t")


class _Layer:
    __slots__ = ("name", "kind", "cin", "cout", "k", "w_t", "bias", "gamma", "beta", "lora", "w_c4", "w_c4_t")


# a frozen forward GEMM B operand: w = the bf16 weights of its member layers stacked along N, K-blocked
# [K/64][N][64] (pcm_bsrc.kblocked), in a storage of its own; members = [(layer, its first row n0)]
Operand = namedtuple("Operand", "w members")


def _stacks(tab):
    """The layers whose frozen weights are stacked along N into ONE forward operand because they read the
    same input and run as one GEMM: [(operand key, kind, member names in row order)] for
      * "qkv": the attn1 q / k / v of every transformer block (key: its to_q);
      * "temb": every resnet's time_emb_proj, which read the same silu(temb) (1 base K entry + one N-ranged
        LoRA entry per layer must fit the K program);
      * "ctx": the cross-attention k / v of ALL transformer blocks, which read the same text context, in
        chunks of at most 11 blocks of one width (22 N-ranged LoRA entries + the base entry <= PCM_MAX_PROG)."""
    names = [n for n, *_ in tab]
    out = [(n, "qkv", [n[:-1] + c for c in "qkv"]) for n in names if n.endswith(".attn1.to_q")]
    temb = [n for n in names if n.endswith(".time_emb_proj")]
    if len(temb) > 23:
        raise ValueError(f"{len(temb)} time_emb_proj layers: the grouped time-embedding GEMM holds at most 23 "
                         f"(PCM_MAX_PROG - 1)")
    out.append(("temb", "temb", temb))
    co = {n: c for n, _, _, c, _ in tab}
    chunks = []
    for n in sorted((n for n in names if n.endswith(".attn2.to_k")), key=co.get):   # stable: one width together
        if not chunks or co[chunks[-1][0]] != co[n] or len(chunks[-1]) == 22:
            chunks.append([])
        chunks[-1] += [n, n[:-1] + "v"]
    return out + [(f"ctx.{c}", "ctx", ch) for c, ch in enumerate(chunks)]


@dataclass
class _Pass:
    """One forward pass: what its primitives read besides their own arguments."""
    lora: bool                              # the LoRA adapters are on
    B: int                                  # samples in the batch
    lb: int                                 # the leading samples that carry the adapter
    plan_b: Optional[int] = None            # a rebuilt block: the merged pass's batch, whose plans it keeps
    st: Optional[torch.Tensor] = None       # silu(temb) [B, C]
    ctx: Optional[torch.Tensor] = None      # text context [B*S, D]
    temb: Optional[tuple] = None            # UNetB200.temb_all: (out_all, T)
    ctxkv: Optional[dict] = None            # UNetB200.ctx_kv_all: {transformer block: (k, v, T)}

    def rows(self, n):
        """Rows / samples of an n-row (batch-major) tensor that belong to the LoRA samples."""
        return n * self.lb // self.B

    def tiling(self, M, N, prog):
        """Tiling keywords of a block's main GEMM.  Empty (ops.gemm picks from M) except in a rebuilt
        block: then the (block_n, ksplit) the merged pass picked for its larger M, since pick_tiling splits
        K by M and the split decides how the fp32 sums round.  The LoRA down-projections already ran on the
        student rows alone and need nothing."""
        if self.plan_b is None:
            return {}
        bn, ks = ops.pick_tiling(M * self.plan_b // self.B, N, sum(e[4] for e in prog))
        return dict(block_n=bn, ksplit=ks)

    def student(self):
        """The pass a checkpointed block of this one is rebuilt in: the student rows of its time embedding,
        context, grouped time_emb_proj output and context k / v, with this pass's launch plans."""
        lb, S = self.lb, self.ctx.shape[0] // self.B
        kv = self.ctxkv and {t: (k[:lb * S], v[:lb * S], T) for t, (k, v, T) in self.ctxkv.items()}
        return _Pass(self.lora, lb, lb, self.B if self.B != lb else None, self.st[:lb], self.ctx[:lb * S],
                     (self.temb[0][:lb], self.temb[1]), kv)


# forward(save=True) for backward(): the block records in forward order, the head GroupNorm's record,
# (student samples, H, W) and the student pass that rebuilds checkpointed blocks (None: no checkpointing)
Saved = namedtuple("Saved", "tape head shape rebuild")


@dataclass
class _Backward:
    """Scratch of one backward() call."""
    wstream: Optional[torch.cuda.Stream] = None  # the weight-gradient side stream (None: none, all in order)
    dkv: dict = field(default_factory=dict)     # per context chunk: the dk / dv matrix of its shape
    keep: list = field(default_factory=list)    # tensors the weight-gradient stream reads (_Side)
    side: list = field(default_factory=list)    # checkpointing: (event, keep) of the last blocks walked


class UNetB200:
    gradient_checkpointing = False

    def __init__(self, cfg: UNetConfig, state_dict, device, need_backward=True, lora=True,
                 gradient_checkpointing=False):
        """gradient_checkpointing: a forward with save=True keeps only the student rows of every block's
        inputs; backward() runs each block's forward again right before its backward (see forward())."""
        self.cfg, self.dev = cfg, device
        self.gradient_checkpointing = gradient_checkpointing
        self.r = check_lora_rank(cfg.lora_rank) if lora else cfg.lora_rank
        self.rc = (self.r + 63) // 64       # 64-wide K chunks / weight-gradient rank slices of one adapter
        self.scale = cfg.lora_scale
        self.layers = {}
        self.has_lora = lora
        tab = layer_table(cfg)
        stacks = _stacks(tab)
        stacked = {n for _, _, names in stacks for n in names}
        # every cross-attention k / v layer, chunk after chunk: one LoRA down-projection serves all chunks
        self._ctx_names = [n for _, kind, names in stacks if kind == "ctx" for n in names]
        master, entries, opnd_total = [], [], 0
        moff = 0
        for name, kind, cin, cout, k in tab:
            L = _Layer()
            L.name, L.kind, L.cin, L.cout, L.k = name, kind, cin, cout, k
            L.w_t = L.bias = L.gamma = L.beta = L.lora = L.w_c4 = L.w_c4_t = None
            if kind in ("gn", "ln"):
                L.gamma = state_dict[name + ".weight"].float().to(device)
                L.beta = state_dict[name + ".bias"].float().to(device)
                self.layers[name] = L
                continue
            W = state_dict[name + ".weight"].float()
            if (name + ".bias") in state_dict:
                L.bias = state_dict[name + ".bias"].float().to(device)
            if name == "conv_in":
                L.w_c4 = W.permute(0, 2, 3, 1).contiguous().to(device=device, dtype=BF16)  # [C][3][3][4]
            elif name == "conv_out":
                L.w_c4_t = W.permute(1, 2, 3, 0).contiguous().to(device=device, dtype=BF16)  # [C][3][3][4]
            elif kind == "conv":
                if need_backward:
                    L.w_t = self._kblocked(W.permute(1, 2, 3, 0).reshape(cin, -1))
            # no input gradient through the (frozen) time embedding, nor per stacked layer: time_emb_proj and
            # the cross-attention k / v read inputs nothing trains, q / k / v run one dgrad over the group
            elif need_backward and name not in stacked and not name.startswith(("time_embedding", "add_embedding")):
                L.w_t = self._kblocked(W.t())
            if lora and is_lora_target(name):
                taps = k * k if kind == "conv" else 1
                A = state_dict[name + ".lora_A.weight"].float()
                Bm = state_dict[name + ".lora_B.weight"].float()
                if A.shape[0] != self.r or Bm.shape[1] != self.r:
                    raise ValueError(f"{name}: the state dict holds a rank-{A.shape[0]} LoRA adapter "
                                     f"(lora_B rank {Bm.shape[1]}), the UNet is configured for rank {self.r}")
                if kind == "conv":
                    A = A.permute(0, 2, 3, 1)
                A = A.reshape(self.r, taps * cin)
                Bm = Bm.reshape(cout, self.r)
                lo = _Lora()
                lo.a_off, lo.b_off = moff, moff + A.numel()
                moff += A.numel() + Bm.numel()
                master += [A.flatten(), Bm.flatten()]
                lo.opnd_off = opnd_total
                opnd_total += 2 * A.numel() + 2 * Bm.numel()
                L.lora = lo
                entries.append((L, taps))
            self.layers[name] = L
        self.lora_layers = [e[0] for e in entries]
        if lora and entries:
            self.lora_master = torch.cat(master).to(device)
            self.lora_grad = torch.zeros_like(self.lora_master)
            self.lora_opnd = torch.empty(opnd_total, device=device, dtype=BF16)
            # operand copies: [A | s*B | (s*B)^T | A^T] per layer; the layers of a stack are laid out
            # kind-major so that their A, s*B and (s*B)^T copies stack into single GEMM operands, and so are
            # the cross-attention k / v layers of ALL chunks: one down-projection serves every chunk
            unit_of = {n: self._ctx_names if kind == "ctx" else names for _, kind, names in stacks for n in names}
            by_name = {L.name: (L, taps) for L, taps in entries}
            units, seen = [], set()
            for L, taps in entries:
                if L.name in seen:
                    continue
                grp = unit_of.get(L.name)
                members = [by_name[n] for n in grp] if grp and all(n in by_name for n in grp) else [(L, taps)]
                seen.update(m[0].name for m in members)
                units.append(members)
            o = 0
            for members in units:
                for kind in ("a_fwd", "sb_fwd", "sb_t", "a_t"):
                    for L, taps in members:
                        n = self.r * taps * L.cin if kind in ("a_fwd", "a_t") else L.cout * self.r
                        setattr(L.lora, "o_" + kind, o)
                        o += n
            assert o == opnd_total
            rows, work = [], 0
            for L, taps in entries:
                lo = L.lora
                na, nb = self.r * taps * L.cin, L.cout * self.r
                a_fwd, sb_fwd, sb_t, a_t = lo.o_a_fwd, lo.o_sb_fwd, lo.o_sb_t, lo.o_a_t
                lo.a_fwd = self.lora_opnd[a_fwd:a_fwd + na].view(self.r, taps * L.cin)
                lo.sb_fwd = self.lora_opnd[sb_fwd:sb_fwd + nb].view(L.cout, self.r)
                lo.sb_t = self.lora_opnd[sb_t:sb_t + nb].view(self.r, L.cout)
                lo.a_t = self.lora_opnd[a_t:a_t + na].view(L.cin, taps * self.r)
                lo.gA = self.lora_grad[lo.a_off:lo.a_off + na].view(self.r, taps * L.cin)
                lo.gB = self.lora_grad[lo.b_off:lo.b_off + nb].view(L.cout, self.r)
                rows.append([lo.a_off, lo.b_off, a_fwd, sb_fwd, sb_t, a_t, L.cin | (taps << 32),
                             L.cout | (self.r << 32), work])
                assert L.cin % 64 == 0 and L.cout % 64 == 0
                # (min(r, 64) x 64) tiles of A, then of B, per 64-rank slice
                work += self.rc * ((taps * L.cin) // 64 + L.cout // 64)
            self.refresh_table = torch.tensor(rows, dtype=torch.int64, device=device)
            self.refresh_work = work
            self.refresh_lora()
        self._build_operands(state_dict, tab, stacks, stacked)
        self._build_groups(state_dict, stacks, need_backward)
        self._build_temb_group(next(names for _, kind, names in stacks if kind == "temb"))
        self._build_ctx_group([(key, names) for key, kind, names in stacks if kind == "ctx"])
        self.saved = None
        # LoRA weight-gradient GEMMs are off the dgrad critical path (they only feed the optimiser):
        # they run on a side stream and fill SMs the main backward chain leaves idle
        use_wstream = torch.device(device).type == "cuda" and need_backward and lora
        self.wstream = torch.cuda.Stream(device=device) if use_wstream else None

    def _kblocked(self, W):
        """bf16 copy of the fp32 [N, K] matrix W on the device, K-blocked [K/64][N][64] (pcm_bsrc.kblocked):
        the operand tile of a K block is one contiguous run in HBM.  Matters for the small-M layers (8x8 /
        16x16 levels, target pass), which stream their weights once per launch: a row-major tile is N
        separate 128-byte segments K*2 bytes apart."""
        return ops.kblock(W.to(device=self.dev, dtype=BF16))

    def _build_operands(self, state_dict, tab, stacks, stacked):
        """self.operands = {key: Operand}: the forward B operand of every GEMM that reads a frozen weight,
        built once from the state dict.  Every Linear / 1x1 / 3x3 layer outside a stack has its own (key:
        the layer name), then come the stacks of _stacks.  conv_in runs its own 4-channel kernel on w_c4."""
        single = [(n, [n]) for n, kind, *_ in tab if kind not in ("gn", "ln") and n != "conv_in" and n not in stacked]
        self.operands = {}
        for key, names in single + [(key, names) for key, _, names in stacks]:
            Ls = [self.layers[n] for n in names]
            rows = []
            for L in Ls:
                W = state_dict[L.name + ".weight"].float()
                rows.append(W.permute(0, 2, 3, 1).reshape(L.cout, -1) if L.kind == "conv" else W)  # [N, taps*cin]
            n0 = [sum(L.cout for L in Ls[:i]) for i in range(len(Ls))]
            self.operands[key] = Operand(self._kblocked(torch.cat(rows)), list(zip(Ls, n0)))

    def _stacked(self, layers, kind, rows, cols):
        """The `kind` ("a_fwd", "sb_fwd", "sb_t") operand copies of `layers`, laid out kind-major next to
        each other in lora_opnd, as ONE [rows, cols] view."""
        o = getattr(layers[0].lora, "o_" + kind)
        v = self.lora_opnd[o:o + rows * cols].view(rows, cols)
        last = getattr(layers[-1].lora, kind)
        assert last.data_ptr() == v.view(-1)[-last.numel():].data_ptr()
        return v

    def _build_groups(self, state_dict, stacks, need_backward):
        """self.groups, keyed by their first layer: the shared-input Linear groups, whose LoRA operand copies
        are viewed as stacks so that their LoRA K blocks enter one GEMM.  The q / k / v of a transformer
        block run forward as ONE GEMM over their stacked operand (N = 3C) and backward as one dgrad GEMM
        over w_t_cat [cin, 3C]; the cross-attention k / v of one block run forward in a context chunk and
        backward only into their LoRA weight gradients."""
        self.groups = {}
        qkv = [(names, need_backward) for _, kind, names in stacks if kind == "qkv"]
        kv = [(names[i:i + 2], False) for _, kind, names in stacks if kind == "ctx" for i in range(0, len(names), 2)]
        for names, dgrad in qkv + kv:
            Ls = [self.layers[n] for n in names]
            assert all(L.bias is None and L.cin == Ls[0].cin and L.cout == Ls[0].cout for L in Ls)
            G = types.SimpleNamespace(names=names, layers=Ls, g=len(Ls), cin=Ls[0].cin, cout=Ls[0].cout)
            G.w_t_cat = None
            if dgrad:       # [cin, g*C]
                G.w_t_cat = self._kblocked(torch.cat([state_dict[n + ".weight"].float() for n in names]).t())
            G.lora = all(L.lora is not None for L in Ls)
            if G.lora:
                r, g = self.r, G.g
                G.a_stack = self._stacked(Ls, "a_fwd", g * r, G.cin)
                G.sb_stack = self._stacked(Ls, "sb_fwd", g * G.cout, r)
                G.sbt_stack = self._stacked(Ls, "sb_t", g * r, G.cout)
            self.groups[names[0]] = G

    def _build_temb_group(self, names):
        """The time-embedding projections, which run as ONE GEMM over the "temb" operand: column offsets,
        bias [sum C_i] and the kind-major LoRA copies A [g*r, temb], s*B [sum C_i, r]."""
        Ls = [self.layers[n] for n in names]
        G = types.SimpleNamespace(names=names, layers=Ls, g=len(Ls), cin=Ls[0].cin)
        assert all(L.cin == G.cin and L.bias is not None for L in Ls)
        G.offs = [0]
        for L in Ls:
            G.offs.append(G.offs[-1] + L.cout)
        G.n_total = G.offs[-1]
        assert G.n_total < 65536
        G.bn = 160 if all(o % 160 == 0 for o in G.offs) else 64
        G.index = {n: i for i, n in enumerate(G.names)}
        G.bias = torch.cat([L.bias for L in Ls]).contiguous()
        G.lora = all(L.lora is not None for L in Ls)
        if G.lora:
            G.a_stack = self._stacked(Ls, "a_fwd", G.g * self.r, G.cin)
            G.sb_stack = self._stacked(Ls, "sb_fwd", G.n_total, self.r)
        self.temb_group = G

    def _lora_down(self, x, a_stack):
        """T = x @ a_stack^T: the LoRA down-projections of several layers that read the same x."""
        T = self._new(x.shape[0], a_stack.shape[0])
        ops.gemm([ops.asrc_mat(x)], [ops.bsrc(a_stack)], [(0, 0, 0, 0, x.shape[1] // 64, 0, 0)], lin=True,
                 M=x.shape[0], N=a_stack.shape[0], out=T)
        return T

    def _stacked_gemm(self, x, w_stack, T, sb_stack, ranges, N, *, block_n, bias=None, dep_a_src=None):
        """out[M, N] = [x | T] @ [w_stack ; sb_stack]^T (+ bias): the frozen weights of several layers stacked
        along N, then one LoRA K entry per layer that reads T columns [t_c0, t_c0 + r) and only feeds that
        layer's output columns [n_lo, n_hi); ranges = [(t_c0, n_lo, n_hi)] (unused when T is None)."""
        srcs, bs = [ops.asrc_mat(x)], [ops.bsrc(w_stack)]
        prog = [(0, 0, 0, 0, x.shape[1] // 64, 0, 0)]
        if T is not None:
            srcs.append(ops.asrc_mat(T))
            bs.append(ops.bsrc(sb_stack))
            prog += [(1, 1, 0, 0, self.rc, t_c0, 0, n_lo, n_hi) for t_c0, n_lo, n_hi in ranges]
        out = self._new(x.shape[0], N)
        ops.gemm(srcs, bs, prog, lin=True, M=x.shape[0], N=N, out=out, bias=bias, block_n=block_n,
                 dep_a_src=dep_a_src)
        return out

    def temb_all(self, P):
        """All time_emb_proj layers of pass P: out[B, sum C_i] = [st | T] @ [W ; N-ranged s*B_i]^T + b.
        Returns (out, T): resnet i uses the column view out[:, offs[i]:offs[i+1]] as its row vector and
        column block i of T for its LoRA weight gradients."""
        G, r, st = self.temb_group, self.r, P.st
        T = self._lora_down(st[:P.rows(st.shape[0])], G.a_stack) if P.lora and G.lora else None
        out = self._stacked_gemm(st, self.operands["temb"].w, T, getattr(G, "sb_stack", None),
                                 [(i * r, G.offs[i], G.offs[i + 1]) for i in range(G.g)], G.n_total,
                                 block_n=G.bn, bias=G.bias)
        return out, T

    def _build_ctx_group(self, chunks):
        """Cross-attention k / v of ALL transformer blocks from the text context (they depend on nothing
        else), chunks = [(operand key, member names)]: A copies of every layer stacked [n_layers*r, ctx_dim]
        for ONE down-projection GEMM, and per chunk the s*B copies stacked like its frozen operand."""
        self.ctx_group = None
        if not chunks:
            return
        names = self._ctx_names
        Ls = [self.layers[n] for n in names]
        assert all(L.bias is None and L.cin == Ls[0].cin for L in Ls)
        CG = types.SimpleNamespace(names=names, cin=Ls[0].cin, nl=len(names), chunks=[], where={})
        CG.lora = all(L.lora is not None for L in Ls)
        if CG.lora:
            CG.a_stack = self._stacked(Ls, "a_fwd", CG.nl * self.r, CG.cin)
        first = 0
        for key, ch_names in chunks:
            blocks = [self.groups[n] for n in ch_names[::2]]
            ch = types.SimpleNamespace(key=key, cout=blocks[0].cout, blocks=blocks, first=first)
            ch.n_total = 2 * ch.cout * len(blocks)
            assert ch.n_total < 65536
            ch.bn = 160 if ch.cout % 160 == 0 else 64
            if CG.lora:
                ch.sb_stack = self._stacked([L for G in blocks for L in G.layers], "sb_fwd", ch.n_total, self.r)
            for j, G in enumerate(blocks):
                CG.where[G.names[0][:-len(".attn2.to_k")]] = (len(CG.chunks), j)
            CG.chunks.append(ch)
            first += len(ch_names)
        self.ctx_group = CG

    def ctx_kv_all(self, P):
        """{transformer block: (k, v, T)} for pass P: k / v are column views [M, C] of the chunk outputs,
        T the block's two columns blocks [Ml, 2r] of the stacked LoRA down-projection (None without LoRA)."""
        CG, r, ctx = self.ctx_group, self.r, P.ctx
        T = self._lora_down(ctx[:P.rows(ctx.shape[0])], CG.a_stack) if P.lora and CG.lora else None
        outs = [self._stacked_gemm(ctx, self.operands[ch.key].w, T, getattr(ch, "sb_stack", None),
                                   [((ch.first + i) * r, i * ch.cout, (i + 1) * ch.cout)
                                    for i in range(2 * len(ch.blocks))], ch.n_total, block_n=ch.bn)
                for ch in CG.chunks]
        kv = {}
        for t, (c, j) in CG.where.items():
            ch, out = CG.chunks[c], outs[c]
            Cc = ch.cout
            Tb = None if T is None else T[:, (ch.first + 2 * j) * r:(ch.first + 2 * j + 2) * r]
            kv[t] = (out[:, 2 * j * Cc:(2 * j + 1) * Cc], out[:, (2 * j + 1) * Cc:(2 * j + 2) * Cc], Tb)
        return kv

    @staticmethod
    def ctx_kv_rows(kv, rows):
        """The leading `rows` context rows of a ctx_kv_all result (k / v only): the student samples'
        projections of the merged pass, reused by the target pass (same context, same weights)."""
        return {t: (k[:rows], v[:rows], None) for t, (k, v, _) in kv.items()}

    class _Side:
        """Run the enclosed launches on the wgrad side stream, ordered after everything enqueued so far
        on the current stream; `keep` tensors stay referenced (bw.keep) until backward() joins the streams."""

        def __init__(self, bw, keep):
            self.bw, self.keep, self.ctx = bw, keep, None

        def __enter__(self):
            bw = self.bw
            if bw.wstream is None:
                return self
            ev = torch.cuda.Event()
            ev.record()
            bw.wstream.wait_event(ev)
            bw.keep.extend(self.keep)
            self.ctx = torch.cuda.stream(bw.wstream)
            self.ctx.__enter__()
            return self

        def __exit__(self, *a):
            if self.ctx is not None:
                self.ctx.__exit__(*a)
            return False

    # ------------------------------------------------------------------------------------
    def refresh_lora(self, master=None):
        """Regenerate the bf16 GEMM operand copies (A, s*B, (s*B)^T, A^T) from the fp32 masters
        (`master`: another flat buffer of the same layout, e.g. an EMA copy for the target pass)."""
        master = self.lora_master if master is None else master
        assert master.numel() == self.lora_master.numel() and master.dtype == torch.float32
        ops._call("pcm_lora_refresh", master.data_ptr(), self.refresh_table.data_ptr(),
                  self.refresh_table.shape[0], self.refresh_work, self.scale, self.lora_opnd.data_ptr())

    def fused_inference_net(self):
        """An inference network over this one's weights with the LoRA fused in (peft `fuse_lora`): no
        backward, no LoRA operands, no tape.  Every operand of self.operands whose layers are LoRA targets
        (single layers, the q/k/v stacks, the time_emb_proj stack, the cross-attention k / v context
        chunks) gets a fused copy in ONE new bf16 buffer, net.fused_weights; net.operands points there.
        Everything else (layers, groups, norms, biases, the other operands) is this network's own.
        Returns (net, fuse_table, fuse_work): fuse_table is the int64 [entries, 8] table of pcm_lora_fuse
        (ops.lora_fuse), one row per LoRA layer: {a_off, b_off, src, dst, n0 | N_total << 32, K | r << 32,
        n, work_begin}."""
        if not self.has_lora:
            raise ValueError("fused_inference_net needs a network built with lora=True")
        net = copy.copy(self)
        for k in ("lora_master", "lora_grad", "lora_opnd", "refresh_table", "refresh_work"):
            net.__dict__.pop(k, None)
        net.has_lora, net.wstream = False, None
        net.gradient_checkpointing, net.lora_layers, net.saved = False, [], None
        fused = {key: op for key, op in self.operands.items() if any(L.lora is not None for L, _ in op.members)}
        net.fused_weights = torch.empty(sum(op.w.numel() for op in fused.values()), device=self.dev, dtype=BF16)
        net.operands = dict(self.operands)
        rows, work, off = [], 0, 0
        for key, (src, members) in fused.items():
            dst = net.fused_weights[off:off + src.numel()].view(src.shape)
            off += src.numel()
            net.operands[key] = Operand(dst, members)
            K, ntot = src.shape[0] * 64, src.shape[1]
            for L, n0 in members:
                taps = L.k * L.k if L.kind == "conv" else 1
                assert L.lora is not None and taps * L.cin == K and L.cout % 64 == 0
                rows.append([L.lora.a_off, L.lora.b_off, src.data_ptr(), dst.data_ptr(), n0 | (ntot << 32),
                             K | (self.r << 32), L.cout, work])
                work += (L.cout // 64) * (K // 64)
        table = torch.tensor(rows, dtype=torch.int64, device=self.dev)
        return net, table, work

    def block_grad_offsets(self):
        """First flat-buffer offset of every UNet block (resnet / transformer / resample conv) that owns
        LoRA layers, ascending - the bucket boundaries of the overlapped gradient all-reduce."""
        offs = {}
        for L in self.lora_layers:
            blk = self._block_of(L.name)
            offs[blk] = min(offs.get(blk, 1 << 62), L.lora.a_off)
        return offs

    @staticmethod
    def _block_of(layer_name):
        parts = layer_name.split(".")
        if parts[0] == "mid_block":
            return ".".join(parts[:3])
        if parts[2] in ("downsamplers", "upsamplers"):
            return ".".join(parts[:5])
        return ".".join(parts[:4])

    def lora_state_dict(self):
        """peft-style tensors (`<module>.lora_A.weight` [r, cin(,k,k)], `.lora_B.weight`)."""
        out = {}
        for L in self.lora_layers:
            lo = L.lora
            taps = L.k * L.k if L.kind == "conv" else 1
            A = self.lora_master[lo.a_off:lo.a_off + self.r * taps * L.cin]
            Bm = self.lora_master[lo.b_off:lo.b_off + L.cout * self.r]
            if L.kind == "conv":
                out[L.name + ".lora_A.weight"] = A.view(self.r, L.k, L.k, L.cin).permute(0, 3, 1, 2).clone()
                out[L.name + ".lora_B.weight"] = Bm.view(L.cout, self.r, 1, 1).clone()
            else:
                out[L.name + ".lora_A.weight"] = A.view(self.r, L.cin).clone()
                out[L.name + ".lora_B.weight"] = Bm.view(L.cout, self.r).clone()
        return out

    def lora_grad_dict(self):
        out = {}
        for L in self.lora_layers:
            lo = L.lora
            if L.kind == "conv":
                out[L.name + ".lora_A.weight"] = lo.gA.view(self.r, L.k, L.k, L.cin).permute(0, 3, 1, 2).clone()
                out[L.name + ".lora_B.weight"] = lo.gB.view(L.cout, self.r, 1, 1).clone()
            else:
                out[L.name + ".lora_A.weight"] = lo.gA.clone()
                out[L.name + ".lora_B.weight"] = lo.gB.clone()
        return out

    # ------------------------------------------------------------------------------------
    # primitive layers (forward)
    # ------------------------------------------------------------------------------------
    def _new(self, *shape, dtype=BF16):
        return torch.empty(*shape, device=self.dev, dtype=dtype)

    def conv3(self, P, name, xs, stride=1, rowvec=None, residual=None, out_fp32=False, save=None):
        """3x3 pad-1 convolution (+LoRA) over NHWC sources xs (channel concat), fused epilogue; appends its
        ConvRec to the list `save`."""
        L = self.layers[name]
        B, H, W, _ = xs[0].shape
        Ho, Wo = H // stride, W // stride
        M, N = B * Ho * Wo, L.cout
        srcs, prog = conv_prog(xs, 3, stride, L.cin)
        bs = [ops.bsrc(self.operands[name].w)]
        T = None
        lbn = P.rows(B)   # samples that carry the LoRA adapter (the leading ones of the batch)
        xl = xs if lbn == B else [x[:lbn] for x in xs]
        if P.lora and L.lora is not None:
            # T = A(x) only for the LoRA samples; the other samples see T rows that TMA zero-fills
            T = self._new(lbn, Ho, Wo, self.r)
            srcs_l, prog_l = (srcs, prog) if lbn == B else conv_prog(xl, 3, stride, L.cin)
            ops.gemm(srcs_l, [ops.bsrc(L.lora.a_fwd)], prog_l, lin=False, M=lbn * Ho * Wo, N=self.r,
                     geo=(Wo, Ho), out=T.view(lbn * Ho * Wo, self.r))
            prog = prog + [(len(srcs), 1, 0, 0, self.rc, 0, 0)]
            srcs = srcs + [ops.asrc_nhwc(T)]
            bs.append(ops.bsrc(L.lora.sb_fwd))
        out = self._new(B, Ho, Wo, N, dtype=torch.float32 if out_fp32 else BF16)
        ops.gemm(srcs, bs, prog, lin=False, M=M, N=N, geo=(Wo, Ho), out=out.view(M, N), bias=L.bias,
                 rowvec=rowvec, residual=None if residual is None else residual.reshape(M, N),
                 round_bf16=out_fp32, dep_a_src=None if T is None else len(srcs) - 1,
                 **P.tiling(M, N, prog))
        if save is not None:
            save.append(ConvRec("conv3", name, xl, T, stride))
        return out

    def linear(self, P, name, xs, residual=None, act=0, save=None):
        """nn.Linear / 1x1 conv over [M, C] matrices xs (channel concat) (+LoRA), fused epilogue; appends its
        LinearRec to the list `save`."""
        L = self.layers[name]
        M, N = xs[0].shape[0], L.cout
        srcs = [ops.asrc_mat(x) for x in xs]
        prog, coff = [], 0
        for si, x in enumerate(xs):
            prog.append((si, 0, 0, 0, x.shape[1] // 64, 0, coff))
            coff += x.shape[1]
        bs = [ops.bsrc(self.operands[name].w)]
        T = None
        Ml = P.rows(M)
        xl = xs if Ml == M else [x[:Ml] for x in xs]
        if P.lora and L.lora is not None:
            T = self._new(Ml, self.r)
            srcs_l = srcs if Ml == M else [ops.asrc_mat(x) for x in xl]
            ops.gemm(srcs_l, [ops.bsrc(L.lora.a_fwd)], prog, lin=True, M=Ml, N=self.r, out=T)
            prog = prog + [(len(srcs), 1, 0, 0, self.rc, 0, 0)]
            srcs = srcs + [ops.asrc_mat(T)]   # Ml rows: tiles past them read zeros (TMA bounds)
            bs.append(ops.bsrc(L.lora.sb_fwd))
        out = self._new(M, N)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=N, out=out, bias=L.bias, residual=residual, act=act,
                 dep_a_src=None if T is None else len(srcs) - 1, **P.tiling(M, N, prog))
        if save is not None:
            save.append(LinearRec("linear", name, xl, T))
        return out

    def linear_group(self, P, lead, x, save=None):
        """The g Linear layers of a shared-input group (attn1 q/k/v, attn2 k/v) as ONE GEMM:
        out[M, g*C] = x @ [W_0; ...; W_g-1]^T, layer i's LoRA up-projection entering as a K block that
        only feeds its own C output columns.  Returns the g column views of out; appends its GroupRec to
        the list `save`."""
        G, r = self.groups[lead], self.r
        g, Cc = G.g, G.cout
        xl = x[:P.rows(x.shape[0])]
        T = self._lora_down(xl, G.a_stack) if P.lora and G.lora else None
        out = self._stacked_gemm(x, self.operands[lead].w, T, getattr(G, "sb_stack", None),
                                 [(i * r, i * Cc, (i + 1) * Cc) for i in range(g)], g * Cc,
                                 block_n=160 if Cc % 160 == 0 else 64, dep_a_src=None if T is None else 1)
        if save is not None:
            save.append(GroupRec("lgroup", lead, xl, T))
        return [out[:, i * Cc:(i + 1) * Cc] for i in range(g)]

    def gn(self, P, name, xs, B, HW, eps, silu, save=None):
        L = self.layers[name]
        C = sum(x.shape[-1] for x in xs)
        out = self._new(B * HW, C)
        stats = self._new(B, self.cfg.norm_num_groups, 2, dtype=torch.float32)
        x2 = xs[1] if len(xs) > 1 else None
        if P.plan_b is None:
            ops.groupnorm_fwd(xs[0], x2, L.gamma, L.beta, eps, silu, out, stats, B, HW, self.cfg.norm_num_groups)
        else:   # a rebuilt block: merge each image's statistics from the merged pass's partition
            ops.groupnorm_fwd_part(xs[0], x2, L.gamma, L.beta, eps, silu, out, stats, B, P.plan_b, HW,
                                   self.cfg.norm_num_groups)
        if save is not None:
            lb = P.rows(B)
            save.append(GNRec("gn", name, xs if lb == B else [x[:lb * HW] for x in xs], stats[:lb], eps, silu, lb, HW))
        return out

    def ln(self, P, name, x, save=None):
        L = self.layers[name]
        out = torch.empty_like(x)
        stats = self._new(x.shape[0], 2, dtype=torch.float32)
        ops.layernorm_fwd(x, L.gamma, L.beta, out, stats)
        if save is not None:
            Ml = P.rows(x.shape[0])
            save.append(LNRec("ln", name, x[:Ml], stats[:Ml]))
        return out

    def attention(self, P, q, k, v, B, Sq, Skv, heads, save=None):
        D = q.shape[1] // heads
        out = self._new(q.shape[0], q.shape[1])
        lse = self._new(B, heads, Sq, dtype=torch.float32)
        ops.attn_fwd(q, k, v, out, lse, B, heads, Sq, Skv, D, D ** -0.5)
        if save is not None:
            lb = P.rows(B)
            save.append(AttnRec("attn", q[:lb * Sq], k[:lb * Skv], v[:lb * Skv], out[:lb * Sq], lse[:lb], lb, Sq, Skv,
                                heads))
        return out

    # ------------------------------------------------------------------------------------
    # blocks (forward): each returns (out, block record)
    # ------------------------------------------------------------------------------------
    def resnet(self, P, p, xs, save):
        """xs: list of NHWC sources (skip concat = 2 sources).  Returns ([B,H,W,Cout], ResnetRec)."""
        B, H, W, _ = xs[0].shape
        HW = H * W
        cin = sum(x.shape[-1] for x in xs)
        cout = self.layers[p + ".conv1"].cout
        flat = [x.view(B * HW, x.shape[-1]) for x in xs]
        s = [] if save else None        # this block's op records
        h = self.gn(P, p + ".norm1", flat, B, HW, 1e-5, True, s)
        norm1 = _last(s)
        G = self.temb_group
        i = G.index[p + ".time_emb_proj"]
        out_all, T_all = P.temb
        # the grouped launch of temb_all computed this layer: its record only names the column block
        temb = TembRec("linear", p + ".time_emb_proj", [P.st[:P.rows(P.st.shape[0])]], T_all, i * self.r)
        h = self.conv3(P, p + ".conv1", [h.view(B, H, W, cin)], rowvec=out_all[:, G.offs[i]:G.offs[i + 1]],
                       save=s)
        conv1 = _last(s)
        h = self.gn(P, p + ".norm2", [h.view(B * HW, cout)], B, HW, 1e-5, True, s)
        norm2 = _last(s)
        sc, shortcut = xs[0], None
        if cin != cout:
            sc = self.linear(P, p + ".conv_shortcut", flat, save=s).view(B, H, W, cout)
            shortcut = _last(s)
        out = self.conv3(P, p + ".conv2", [h.view(B, H, W, cout)], residual=sc, save=s)
        return out, ResnetRec(p, norm1, temb, conv1, norm2, shortcut, _last(s), takes_skip=len(xs) == 2)

    def _level_of(self, name):
        """Resolution level of a block name (selects transformer depth and head count)."""
        nb = len(self.cfg.block_out_channels)
        parts = name.split(".")
        if parts[0] == "mid_block":
            return nb - 1
        i = int(parts[1])
        return i if parts[0] == "down_blocks" else nb - 1 - i

    def transformer(self, P, p, x, save):
        """Transformer2DModel: GN -> proj_in -> depth x BasicTransformerBlock -> proj_out -> + residual.
        proj_in / proj_out are 1x1 convolutions (SD1.5) or nn.Linear (SDXL, use_linear_projection):
        on NHWC tokens both are the same GEMM."""
        B, H, W, C = x.shape
        S, M = H * W, B * H * W
        level = self._level_of(p)
        heads = self.cfg.heads(level)
        xf = x.view(M, C)
        s = [] if save else None        # this block's op records
        g = self.gn(P, p + ".norm", [xf], B, S, 1e-6, False, s)
        norm = _last(s)
        h = self.linear(P, p + ".proj_in", [g], save=s)
        proj_in = _last(s)
        blocks = []
        for d in range(self.cfg.depth(level)):
            t = p + f".transformer_blocks.{d}"
            b = [] if save else None    # the op records of one transformer block, in TBlockRec order
            n = self.ln(P, t + ".norm1", h, b)
            q, k, v = self.linear_group(P, t + ".attn1.to_q", n, save=b)
            a = self.attention(P, q, k, v, B, S, S, heads, b)
            h = self.linear(P, t + ".attn1.to_out.0", [a], residual=h, save=b)
            n = self.ln(P, t + ".norm2", h, b)
            q = self.linear(P, t + ".attn2.to_q", [n], save=b)
            k, v, Tkv = P.ctxkv[t]
            if save:    # k / v came from the context chunks of ctx_kv_all; Tkv is this block's window of T
                b.append(GroupRec("lgroup", t + ".attn2.to_k", P.ctx[:P.rows(P.ctx.shape[0])], Tkv))
            a = self.attention(P, q, k, v, B, S, P.ctx.shape[0] // B, heads, b)
            h = self.linear(P, t + ".attn2.to_out.0", [a], residual=h, save=b)
            n = self.ln(P, t + ".norm3", h, b)
            u = self.linear(P, t + ".ff.net.0.proj", [n], save=b)
            gg = self._new(M, u.shape[1] // 2)
            ops.geglu_fwd(u, gg)
            if save:
                b.append(GegluRec("geglu", u[:P.rows(M)]))
            h = self.linear(P, t + ".ff.net.2", [gg], residual=h, save=b)
            blocks.append(TBlockRec._make(b) if save else None)
        out = self.linear(P, p + ".proj_out", [h], residual=xf, save=s)
        return out.view(B, H, W, C), TransformerRec(p, norm, proj_in, blocks, _last(s))

    def resample(self, P, name, x, save, up):
        """Downsampler (stride-2 convolution) or upsampler (nearest 2x, then the convolution)."""
        s = [] if save else None
        if not up:
            out = self.conv3(P, name, [x], stride=2, save=s)
        else:
            B, H, W, C = x.shape
            xu = self._new(B, 2 * H, 2 * W, C)
            ops.upsample2x_fwd(x, xu)
            out = self.conv3(P, name, [xu], save=s)
        return out, ResampleRec(name, _last(s), up)

    def _block(self, kind, name, xs, P, save, up=False):
        """One block's forward in pass P: (out, record)."""
        if kind == "resnet":
            return self.resnet(P, name, xs, save)
        if kind == "transformer":
            return self.transformer(P, name, xs[0], save)
        return self.resample(P, name, xs[0], save, up)

    def forward(self, sample, timesteps, ctx, lora=True, save=False, lora_batch=None, added_cond=None,
                ctx_kv=None):
        """sample: fp32 [B,H,W,4] NHWC; timesteps: int64 [B]; ctx: bf16 [B*77, D].
        added_cond (SDXL `added_cond_kwargs`, train_pcm_lora_sdxl_adv.py:1094-1133): (text_embeds bf16
        [B, text_embed_dim], time_ids int64 [B, 6]).
        Returns eps fp32 [B,H,W,4] (values rounded to bf16 like the autocast output).

        lora_batch = b < B runs ONE pass in which only the first b samples carry the LoRA adapter
        (student) and the rest see the frozen base weights (teacher): the adapter's T = A(x) is computed
        for the leading rows only and the fused LoRA K-block reads zeros for the others.  The tape then
        holds views of the first b samples, so backward() is the student's backward.

        With gradient_checkpointing, save=True keeps a CheckpointRec per block instead: owned copies of
        the student rows of the block's inputs (one copy per tensor: a down-path output that is the next
        block's input and a skip is kept once), so the merged pass's activations and every block-internal
        tensor are freed as the forward proceeds.  The student pass (the student rows of the pass's time-
        embedding and context projections, small) stays referenced, and the head's GroupNorm record keeps a
        copy of its student rows.  backward() then rebuilds one block's full record at a time."""
        cfg = self.cfg
        lora = lora and self.has_lora
        B, H, W, _ = sample.shape
        P = _Pass(lora, B, lora_batch if (lora and lora_batch) else B, ctx=ctx)
        c0 = cfg.block_out_channels[0]
        emb = self._new(B, c0)
        ops.timestep_embed(timesteps, emb)
        # the time and added embeddings are no LoRA targets: P.lora leaves them frozen
        hemb = self.linear(P, "time_embedding.linear_1", [emb], act=1)
        if not cfg.addition_embed:
            P.st = self.linear(P, "time_embedding.linear_2", [hemb], act=1)  # silu(temb)
        else:
            # "text_time": emb = time_embedding(t) + add_embedding(cat[text_embeds, sinusoid(time_ids)]);
            # every consumer takes silu(emb): the sum and the SiLU run in the last GEMM's epilogue
            if added_cond is None:
                raise ValueError("this UNet needs added_cond = (text_embeds, time_ids) (addition_embed_type text_time)")
            text_embeds, time_ids = added_cond
            temb = self.linear(P, "time_embedding.linear_2", [hemb])
            tid = self._new(B * cfg.num_time_ids, cfg.addition_time_embed_dim)
            ops.timestep_embed(time_ids.reshape(-1), tid)
            add_in = torch.cat([text_embeds.to(BF16), tid.view(B, -1)], dim=1).contiguous()  # [B, 2816] glue
            ah = self.linear(P, "add_embedding.linear_1", [add_in], act=1)
            P.st = self.linear(P, "add_embedding.linear_2", [ah], residual=temb, act=1)
        P.temb = self.temb_all(P)
        # cross-attention k / v of every block: given (ctx_kv: another pass of this step already projected
        # the same context with the same weights) or computed here in a few grouped GEMMs
        if ctx_kv is not None:
            assert not save
            P.ctxkv = ctx_kv
        elif self.ctx_group is not None:
            P.ctxkv = self.ctx_kv_all(P)
        x = self._new(B, H, W, c0)
        Lci = self.layers["conv_in"]
        ops.conv3x3_c4(sample, Lci.w_c4, Lci.bias, x, sgn=1, round_in=True)
        tape, skips = [], [x]       # tape: the block records in forward order
        ck = save and self.gradient_checkpointing
        lb = P.lb
        copies = {}                 # checkpointing: id of a block input -> (weak reference, its copy)

        def student_rows(xs):
            out = []
            for t in xs:
                hit = copies.get(id(t))
                if hit is None or hit[0]() is not t:
                    hit = (weakref.ref(t), t if lb == B else t[:lb].clone())
                    copies[id(t)] = hit
                out.append(hit[1])
            return out

        def run(kind, name, xs, up=False):
            if ck:
                tape.append(CheckpointRec(kind, name, student_rows(xs), len(xs) == 2, up))
                return self._block(kind, name, xs, P, False, up)[0]
            out, rec = self._block(kind, name, xs, P, save, up)
            tape.append(rec)
            return out

        def push(x):                # the last block's output x becomes a skip input of the up path
            tape[-1].pushes_skip = True
            skips.append(x)

        nb = len(cfg.block_out_channels)
        for i in range(nb):
            for j in range(cfg.layers_per_block):
                x = run("resnet", f"down_blocks.{i}.resnets.{j}", [x])
                if cfg.down_attn[i]:
                    x = run("transformer", f"down_blocks.{i}.attentions.{j}", [x])
                push(x)
            if i < nb - 1:
                x = run("resample", f"down_blocks.{i}.downsamplers.0.conv", [x])
                push(x)
        x = run("resnet", "mid_block.resnets.0", [x])
        x = run("transformer", "mid_block.attentions.0", [x])
        x = run("resnet", "mid_block.resnets.1", [x])
        for i in range(nb):
            for j in range(cfg.layers_per_block + 1):
                x = run("resnet", f"up_blocks.{i}.resnets.{j}", [x, skips.pop()])
                if cfg.up_attn[i]:
                    x = run("transformer", f"up_blocks.{i}.attentions.{j}", [x])
            if i < nb - 1:
                x = run("resample", f"up_blocks.{i}.upsamplers.0.conv", [x], up=True)
        Bx, Hx, Wx, Cx = x.shape
        head = [] if save else None
        g = self.gn(P, "conv_norm_out", [x.view(Bx * Hx * Wx, Cx)], Bx, Hx * Wx, 1e-5, True, head)
        eps = self.conv3(P, "conv_out", [g.view(Bx, Hx, Wx, Cx)], out_fp32=True)
        if save:
            h = head[0]
            if ck and lb != B:      # the student rows are views of the merged pass's last activation
                h = h._replace(xs=[t.clone() for t in h.xs], stats=h.stats.clone())
            self.saved = Saved(tape, h, (lb, H, W), P.student() if ck else None)
        return eps

    def saved_ctx_kv(self):
        """{transformer block: (k, v, T)}: the student rows of the context k / v of the pass forward(save=True)
        saved, which a later pass of the student on the same context takes (forward(ctx_kv=...))."""
        tape, _, _, rebuild = self.saved
        if rebuild is not None:
            return rebuild.ctxkv
        return {f"{blk.name}.transformer_blocks.{d}": (b.attn2.k, b.attn2.v, b.attn2_kv.T)
                for blk in tape if isinstance(blk, TransformerRec) for d, b in enumerate(blk.blocks)}

    # ------------------------------------------------------------------------------------
    # backward primitives
    # ------------------------------------------------------------------------------------
    def _lora_wgrads(self, L, M, dy, T, dt, P_list, t_c0=0, dt_c0=0, lin=True, geo=(1, 1)):
        """LoRA weight gradients of layer L (called inside _Side): dB += s * dy^T T[:, t_c0:t_c0+r] and
        dA += dt[:, dt_c0:dt_c0+r]^T x for each (x, taps, tap offsets) of P_list.  dy, T, dt: A-operand
        sources with M rows."""
        lo, r = L.lora, self.r
        if r % 64:
            # the kernel's rank slice is min(64, q.C - q_c0) wide: end stacked T / dT views at this
            # layer's last rank column so that no slice reaches into the next layer's columns
            T, dt = ops.asrc_cols(T, t_c0 + r), ops.asrc_cols(dt, dt_c0 + r)
        # one launch per 64-rank slice j (r > 64): ranks [64j, 64j + 64) of gB's rows / gA's rows
        for j in range(self.rc):
            ops.wgrad(dy, T, lo.gB[:, 64 * j:], lin=True, M=M, os_row=r, os_col=1, alpha=self.scale,
                      q_c0=t_c0 + 64 * j)
        for j in range(self.rc):
            for psrc, taps, offs in P_list:
                ops.wgrad(psrc, dt, lo.gA[64 * j:], lin=lin, M=M, geo=geo, taps=taps, tap_off=offs, os_row=1,
                          os_col=lo.gA.shape[1], q_c0=dt_c0 + 64 * j)

    def linear_bwd(self, bw, rec, dy, need_dx=True, t_c0=0):
        """rec: LinearRec (or TembRec, whose block of T starts at column t_c0).  Returns dx [M, cin_total]
        (or None)."""
        L = self.layers[rec.name]
        M = dy.shape[0]
        srcs = [ops.asrc_mat(dy)]
        dt = None
        if rec.T is not None:
            dt = self._new(M, self.r)
            ops.gemm([ops.asrc_mat(dy)], [ops.bsrc(L.lora.sb_t)], [(0, 0, 0, 0, L.cout // 64, 0, 0)],
                     lin=True, M=M, N=self.r, out=dt)
            P_list, coff = [], 0
            for x in rec.xs:
                P_list.append((ops.asrc_mat(x), ((0, 0),), (coff,)))
                coff += x.shape[1]
            with UNetB200._Side(bw, (dy, rec.T, dt, *rec.xs)):
                self._lora_wgrads(L, M, ops.asrc_mat(dy), ops.asrc_mat(rec.T), ops.asrc_mat(dt), P_list,
                                  t_c0=t_c0)
        if not need_dx:
            return None
        prog = [(0, 0, 0, 0, L.cout // 64, 0, 0)]
        bs = [ops.bsrc(L.w_t)]
        if dt is not None:
            srcs.append(ops.asrc_mat(dt))
            bs.append(ops.bsrc(L.lora.a_t))
            prog.append((1, 1, 0, 0, self.rc, 0, 0))
        dx = self._new(M, L.cin)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=L.cin, out=dx, dep_a_src=None if dt is None else 1)
        return dx

    def linear_group_bwd(self, bw, rec, dpk, need_dx=True):
        """rec: GroupRec ("lgroup", lead, x, T); dpk [M, g*C] = the g output gradients side by side.
        Returns dx [M, cin] (or None): ONE dgrad GEMM over K = g*C (+ the g LoRA blocks)."""
        _, lead, x, T = rec
        G = self.groups[lead]
        g, Cc, r = G.g, G.cout, self.r
        M = dpk.shape[0]
        dT = None
        if T is not None:
            dT = self._new(M, g * r)
            if r % 32 == 0:
                # one GEMM, layer i's K range feeding its own N range [i*r, (i+1)*r): block_n must divide r
                prog = [(0, 0, 0, 0, Cc // 64, i * Cc, 0, i * r, (i + 1) * r) for i in range(g)]
                ops.gemm([ops.asrc_mat(dpk)], [ops.bsrc(G.sbt_stack)], prog, lin=True, M=M, N=g * r, out=dT,
                         block_n=64 if r % 64 == 0 else 32)
            else:
                # N ranges that no block_n can align to: one GEMM per layer into its columns of dT
                for i in range(g):
                    ops.gemm([ops.asrc_mat(dpk)], [ops.bsrc(G.sbt_stack[i * r:(i + 1) * r])],
                             [(0, 0, 0, 0, Cc // 64, i * Cc, 0)], lin=True, M=M, N=r, out=dT[:, i * r:(i + 1) * r])
            with UNetB200._Side(bw, (dpk, T, dT, x)):
                for i, L in enumerate(G.layers):
                    self._lora_wgrads(L, M, ops.asrc_mat(dpk[:, i * Cc:(i + 1) * Cc]), ops.asrc_mat(T),
                                      ops.asrc_mat(dT), [(ops.asrc_mat(x), ((0, 0),), (0,))],
                                      t_c0=i * r, dt_c0=i * r)
        if not need_dx:
            return None
        srcs, bs = [ops.asrc_mat(dpk)], [ops.bsrc(G.w_t_cat)]
        prog = [(0, 0, 0, 0, g * Cc // 64, 0, 0)]
        if dT is not None:
            srcs.append(ops.asrc_mat(dT))
            for i, L in enumerate(G.layers):
                bs.append(ops.bsrc(L.lora.a_t))
                prog.append((1, 1 + i, 0, 0, self.rc, i * r, 0))
        dx = self._new(M, G.cin)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=G.cin, out=dx, dep_a_src=None if dT is None else 1)
        return dx

    def conv3_bwd(self, bw, rec, dy, need_dx=True):
        """rec: ConvRec; dy [B,Ho,Wo,N].  Returns dx [B,H,W,cin_total] (or None)."""
        L = self.layers[rec.name]
        B, Ho, Wo, N = dy.shape
        M = B * Ho * Wo
        geo = (Wo, Ho)
        dy_m = dy.view(M, N)
        dt = None
        if rec.T is not None:
            dt = self._new(B, Ho, Wo, self.r)
            ops.gemm([ops.asrc_mat(dy_m)], [ops.bsrc(L.lora.sb_t)], [(0, 0, 0, 0, N // 64, 0, 0)],
                     lin=True, M=M, N=self.r, out=dt.view(M, self.r))
            if rec.stride == 1:
                P_list, coff = [], 0
                for x in rec.xs:
                    P_list.append((ops.asrc_nhwc(x), TAPS3, [t * L.cin + coff for t in range(9)]))
                    coff += x.shape[-1]
            else:
                # parity plane (p, q) of x meets the kernel rows of _S2_PLANE[p] and columns of _S2_PLANE[q]
                x = rec.xs[0]
                P_list = [(ops.asrc_nhwc(x[:, p::2, q::2, :]),
                           [(sw, sh) for kh, sh in _S2_PLANE[p] for kw, sw in _S2_PLANE[q]],
                           [(kh * 3 + kw) * L.cin for kh, _ in _S2_PLANE[p] for kw, _ in _S2_PLANE[q]])
                          for p in range(2) for q in range(2)]
            with UNetB200._Side(bw, (dy, rec.T, dt, rec.xs)):
                self._lora_wgrads(L, M, ops.asrc_mat(dy_m), ops.asrc_mat(rec.T.view(M, self.r)),
                                  ops.asrc_nhwc(dt), P_list, lin=False, geo=geo)
        if not need_dx:
            return None
        cin = L.cin
        if rec.stride == 1:
            srcs, bs = [ops.asrc_nhwc(dy)], [ops.bsrc(L.w_t)]
            prog = [(0, 0, -dw, -dh, N // 64, 0, t * N) for t, (dw, dh) in enumerate(TAPS3)]
            if dt is not None:
                srcs.append(ops.asrc_nhwc(dt))
                bs.append(ops.bsrc(L.lora.a_t))
                prog += [(1, 1, -dw, -dh, self.rc, 0, t * self.r) for t, (dw, dh) in enumerate(TAPS3)]
            dx = self._new(B, Ho, Wo, cin)
            ops.gemm(srcs, bs, prog, lin=False, M=M, N=cin, geo=geo, out=dx.view(M, cin),
                     dep_a_src=None if dt is None else 1)
            return dx
        # stride 2: one launch per parity plane of dx; x row 2i'+p receives dy row i'-sh through each
        # kernel row (kh, sh) of _S2_PLANE[p] (and likewise for columns)
        H, W = 2 * Ho, 2 * Wo
        dx = self._new(B, H, W, cin)
        for p in range(2):
            for q in range(2):
                taps = [(kh * 3 + kw, -sw, -sh) for kh, sh in _S2_PLANE[p] for kw, sw in _S2_PLANE[q]]
                srcs, bs = [ops.asrc_nhwc(dy)], [ops.bsrc(L.w_t)]
                prog = [(0, 0, dw, dh, N // 64, 0, t * N) for t, dw, dh in taps]
                if dt is not None:
                    srcs.append(ops.asrc_nhwc(dt))
                    bs.append(ops.bsrc(L.lora.a_t))
                    prog += [(1, 1, dw, dh, self.rc, 0, t * self.r) for t, dw, dh in taps]
                plane = dx[:, p::2, q::2, :]
                ops.gemm(srcs, bs, prog, lin=False, M=M, N=cin, geo=geo, out=plane,
                         out_strides=(plane.stride(2), plane.stride(1), plane.stride(0)), epi=(Wo, Wo * Ho),
                         dep_a_src=1 if (dt is not None and p == 0 and q == 0) else None)
        return dx

    def gn_bwd(self, rec, dy, add=None, colsum=None):
        L = self.layers[rec.name]
        xs = rec.xs
        dx1 = torch.empty_like(xs[0])
        dx2 = torch.empty_like(xs[1]) if len(xs) > 1 else None
        red = self._new(rec.B, self.cfg.norm_num_groups, 2, dtype=torch.float32)
        ops.groupnorm_bwd(dy, xs[0], xs[1] if len(xs) > 1 else None, L.gamma, L.beta, rec.eps, rec.silu,
                          rec.stats, red, add, dx1, dx2, rec.B, rec.HW, self.cfg.norm_num_groups, colsum=colsum)
        return dx1, dx2

    def ln_bwd(self, rec, dy, add=None):
        dx = torch.empty_like(rec.x)
        ops.layernorm_bwd(dy, rec.x, self.layers[rec.name].gamma, rec.stats, add, dx)
        return dx

    def attn_bwd(self, bw, rec, dout):
        q, k, v, Hh = rec.q, rec.k, rec.v, rec.heads
        D = q.shape[1] // Hh
        Cc = q.shape[1]
        if q.stride(0) == 3 * Cc:     # self-attention: q/k/v are column views of one [M, 3C] matrix
            pk = self._new(q.shape[0], 3 * Cc)
            dq, dk, dv = pk[:, :Cc], pk[:, Cc:2 * Cc], pk[:, 2 * Cc:]
        else:
            # cross-attention, k/v are column windows of a context chunk [B*77, sum 2C] (ctx_kv_all):
            # dk/dv go to the same window of a gradient matrix of that shape (the attention kernels
            # address k and dk with one row stride); one matrix per chunk and backward pass
            ld, col0 = k.stride(0), k.storage_offset() % k.stride(0)
            assert v.stride(0) == ld and v.storage_offset() == k.storage_offset() + Cc
            dq = self._new(q.shape[0], Cc)
            key = (k.untyped_storage().data_ptr(), ld)
            if key not in bw.dkv:
                bw.dkv[key] = self._new(k.shape[0], ld)
            pk = bw.dkv[key][:, col0:col0 + 2 * Cc]
            dk, dv = pk[:, :Cc], pk[:, Cc:]
        delta = torch.empty_like(rec.lse)
        ops.attn_bwd(q, k, v, rec.out, dout, rec.lse, delta, dq, dk, dv, rec.B, Hh, rec.Sq, rec.Skv, D, D ** -0.5)
        return dq, pk

    # ------------------------------------------------------------------------------------
    # block backward
    # ------------------------------------------------------------------------------------
    def resnet_bwd(self, bw, blk, dout, need_dx=True):
        """dout [B,H,W,Cout].  Returns the gradients (NHWC) of the input and of the skip source (None
        without a skip), or (None, None) without need_dx."""
        B, H, W, cout = dout.shape
        M = B * H * W
        dh2 = self.conv3_bwd(bw, blk.conv2, dout)                      # grad wrt silu(gn2(h1))
        # grad wrt h1 [M, cout]; its per-image column sums (= d tproj[b, n], the time-embedding
        # branch) are accumulated by the same kernel
        cs32 = self._new(B, cout, dtype=torch.float32)
        dh1, _ = self.gn_bwd(blk.norm2, dh2.view(M, cout), colsum=cs32)
        # the time-embedding branch ends in LoRA weight gradients only: all of it on the side stream
        with UNetB200._Side(bw, (cs32,)):
            drow = self._new(B, cout)
            ops.cast_f32_bf16(cs32, drow)
            bw.keep.append(drow)
            self.linear_bwd(bw, blk.temb, drow, need_dx=False, t_c0=blk.temb.t_c0)
        dh = self.conv3_bwd(bw, blk.conv1, dh1.view(B, H, W, cout), need_dx=need_dx)
        dsc = dout.view(M, cout)
        if blk.shortcut is not None:
            dsc = self.linear_bwd(bw, blk.shortcut, dsc, need_dx=need_dx)
        if not need_dx:
            return None, None
        dx1, dx2 = self.gn_bwd(blk.norm1, dh.view(M, -1), add=dsc)
        return dx1.view(B, H, W, -1), None if dx2 is None else dx2.view(B, H, W, -1)

    def transformer_bwd(self, bw, blk, dout):
        """dout [B,H,W,C]; returns dx [B,H,W,C]."""
        B, H, W, C = dout.shape
        M = B * H * W
        do = dout.view(M, C)
        dh = self.linear_bwd(bw, blk.proj_out, do)
        for b in reversed(blk.blocks):
            dh3 = dh
            dgg = self.linear_bwd(bw, b.ff_out, dh3)
            du = torch.empty_like(b.geglu.u)
            ops.geglu_bwd(dgg, b.geglu.u, du)
            dn3 = self.linear_bwd(bw, b.ff_in, du)
            dh2 = self.ln_bwd(b.norm3, dn3, add=dh3)
            da2 = self.linear_bwd(bw, b.attn2_out, dh2)
            dq2, dkv2 = self.attn_bwd(bw, b.attn2, da2)
            with UNetB200._Side(bw, (dkv2,)):     # feeds weight gradients only: off the dgrad chain
                self.linear_group_bwd(bw, b.attn2_kv, dkv2, need_dx=False)
            dn2 = self.linear_bwd(bw, b.attn2_q, dq2)
            dh1 = self.ln_bwd(b.norm2, dn2, add=dh2)
            da1 = self.linear_bwd(bw, b.attn1_out, dh1)
            _, dqkv = self.attn_bwd(bw, b.attn1, da1)
            dn1 = self.linear_group_bwd(bw, b.attn1_qkv, dqkv)
            dh = self.ln_bwd(b.norm1, dn1, add=dh1)
        dg = self.linear_bwd(bw, blk.proj_in, dh)
        dx, _ = self.gn_bwd(blk.norm, dg, add=do)
        return dx.view(B, H, W, C)

    def resample_bwd(self, bw, blk, dout):
        dx = self.conv3_bwd(bw, blk.conv, dout)
        if not blk.up:
            return dx
        B, H, W, C = dx.shape
        d = self._new(B, H // 2, W // 2, C)
        ops.upsample2x_bwd(dx, d)
        return d

    def backward(self, d_eps, grad_ready=None):
        """d_eps: fp32 [B,H,W,4] gradient of the loss w.r.t. the student epsilon.
        Accumulates LoRA gradients into self.lora_grad (caller zeroes it between steps).
        grad_ready(offset): called (on the weight-gradient stream) after each block's backward with
        the flat-buffer offset from which every gradient element is final."""
        tape, head, (B, H, W), rebuild = self.saved
        bw = _Backward(self.wstream)
        boffs = self.block_grad_offsets() if grad_ready is not None else None
        Lco = self.layers["conv_out"]
        c0 = Lco.cin
        dg = self._new(B, H, W, c0)
        ops.conv3x3_c4(d_eps, Lco.w_c4_t, None, dg, sgn=-1, round_in=False)
        d, _ = self.gn_bwd(head, dg.view(B * H * W, c0))
        d = d.view(B, H, W, c0)
        dskips = []     # gradients of the up path's skip inputs; the last one left (conv_in's output) is unused
        done = None     # the block walked before the current one
        for i in reversed(range(len(tape))):
            blk = tape[i]
            if blk.pushes_skip:
                d = ops.add_bf16(d, dskips.pop(), torch.empty_like(d))
            # the block walked before has been fully enqueued by now: its gradients are final once the
            # weight-gradient stream drains
            if grad_ready is not None and boffs.get(done) is not None:
                with UNetB200._Side(bw, ()):
                    grad_ready(boffs[done])
            if isinstance(blk, CheckpointRec):
                # its forward once more, on the saved student rows with the merged pass's launch plans: every
                # tensor of the record is bitwise the one the stored tape would hold
                tape[i] = None              # the rebuilt record holds what the backward still reads
                blk = self._block(blk.kind, blk.name, blk.xs, rebuild, True, blk.up)[1]
            if isinstance(blk, ResnetRec):
                d, dskip = self.resnet_bwd(bw, blk, d, need_dx=i > 0)
                if blk.takes_skip:
                    dskips.append(dskip)
            elif isinstance(blk, TransformerRec):
                d = self.transformer_bwd(bw, blk, d)
            else:
                d = self.resample_bwd(bw, blk, d)
            done = blk.name
            if rebuild is not None:
                self._release_side(bw)
        if grad_ready is not None:
            with UNetB200._Side(bw, ()):
                grad_ready(0)
        if bw.wstream is not None:
            torch.cuda.current_stream().wait_stream(bw.wstream)
        self.saved = None

    def _release_side(self, bw):
        """Checkpointing: the tensors the weight-gradient stream reads stay referenced (_Side keeps them)
        until that stream is done with them.  Joining the streams after every block would serialise the
        weight gradients with the backward chain, so release them one block late: the current stream
        waits for the side work of the block walked before this one, which has had a whole block's
        backward to finish, and then drops its tensors."""
        if bw.wstream is None:
            return
        ev = torch.cuda.Event()
        ev.record(bw.wstream)
        bw.side.append((ev, bw.keep))
        bw.keep = []
        if len(bw.side) > 1:
            ev, _ = bw.side.pop(0)
            torch.cuda.current_stream().wait_event(ev)
