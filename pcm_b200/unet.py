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
import types
import weakref
from collections import namedtuple
from dataclasses import dataclass
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
    __slots__ = ("name", "kind", "cin", "cout", "k", "w_fwd", "w_t", "bias", "gamma", "beta", "lora",
                 "w_c4", "w_c4_t")


class UNetB200:
    gradient_checkpointing = False
    _plan_b = None

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
        # every resnet's time_emb_proj reads the same silu(temb): one grouped GEMM per pass
        # (1 base K entry + one N-ranged LoRA entry per layer must fit the K program)
        self._temb_names = [n for n, *_ in tab if n.endswith(".time_emb_proj")]
        if len(self._temb_names) > 23:
            raise ValueError(f"{len(self._temb_names)} time_emb_proj layers: the grouped time-embedding GEMM "
                             f"holds at most 23 (PCM_MAX_PROG - 1)")
        # every cross-attention k / v projection reads the same text context: a few grouped GEMMs per
        # pass (chunks of <= 11 transformer blocks of one width, _build_ctx_group) instead of one per block
        self._ctx_names = [n for n, *_ in tab if n.endswith((".attn2.to_k", ".attn2.to_v"))]
        _co = {n: co for n, _, _, co, _ in tab}
        self._ctx_names.sort(key=lambda n: _co[n])        # stable: blocks of one width become neighbours
        master, entries, opnd_total = [], [], 0
        moff = 0
        no_dgrad = ("attn2.to_k", "attn2.to_v", "time_emb_proj")
        for name, kind, cin, cout, k in tab:
            L = _Layer()
            L.name, L.kind, L.cin, L.cout, L.k = name, kind, cin, cout, k
            L.w_fwd = L.w_t = L.bias = L.gamma = L.beta = L.lora = L.w_c4 = L.w_c4_t = None
            if kind in ("gn", "ln"):
                L.gamma = state_dict[name + ".weight"].float().to(device)
                L.beta = state_dict[name + ".bias"].float().to(device)
                self.layers[name] = L
                continue
            W = state_dict[name + ".weight"].float()
            if (name + ".bias") in state_dict:
                L.bias = state_dict[name + ".bias"].float().to(device)
            if kind == "conv":
                if name == "conv_in":
                    L.w_c4 = W.permute(0, 2, 3, 1).contiguous().to(device=device, dtype=BF16)  # [C][3][3][4]
                else:
                    L.w_fwd = W.permute(0, 2, 3, 1).reshape(cout, -1).contiguous().to(device=device, dtype=BF16)
                    if name == "conv_out":
                        L.w_c4_t = W.permute(1, 2, 3, 0).contiguous().to(device=device, dtype=BF16)  # [C][3][3][4]
                    elif need_backward:
                        L.w_t = W.permute(1, 2, 3, 0).reshape(cin, -1).contiguous().to(device=device, dtype=BF16)
            else:
                L.w_fwd = W.contiguous().to(device=device, dtype=BF16)
                if need_backward and not name.endswith(no_dgrad) and \
                        not name.startswith(("time_embedding", "add_embedding")):
                    L.w_t = W.t().contiguous().to(device=device, dtype=BF16)
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
            # operand copies: [A | s*B | (s*B)^T | A^T] per layer; the layers of a shared-input group
            # (attn1 q/k/v, attn2 k/v) are laid out kind-major so that their A, s*B and (s*B)^T
            # copies stack into single GEMM operands
            by_name = {L.name: (L, taps) for L, taps in entries}
            units, seen = [], set()
            for L, taps in entries:
                if L.name in seen:
                    continue
                grp = self._unit_of(L.name)
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
        self._build_groups(need_backward)
        self._build_temb_group()
        self._build_ctx_group()
        self._block_weights()
        self.saved = None
        self._temb = None
        self._ctxkv = self.last_ctx_kv = None
        self._dkv_chunks = {}
        self._lb = (1, 1)
        # while backward() rebuilds a checkpointed block: the batch of the merged pass that first ran it,
        # whose launch plans the rebuild keeps (_merged_tiling, gn)
        self._plan_b = None
        # LoRA weight-gradient GEMMs are off the dgrad critical path (they only feed the optimiser):
        # they run on a side stream and fill SMs the main backward chain leaves idle
        self.use_wstream = torch.device(device).type == "cuda" and need_backward and lora
        self.wstream = torch.cuda.Stream(device=device) if self.use_wstream else None
        self._keep = []

    _GROUPS = ((".attn1.to_q", (".attn1.to_q", ".attn1.to_k", ".attn1.to_v")),
               (".attn2.to_k", (".attn2.to_k", ".attn2.to_v")))

    def _group_of(self, name):
        """Names of the shared-input Linear group `name` belongs to (attn1 q/k/v, attn2 k/v, all
        time_emb_proj layers), or None."""
        if name.endswith(".time_emb_proj"):
            return self._temb_names
        for _, sufs in self._GROUPS:
            for suf in sufs:
                if name.endswith(suf):
                    return [name[:-len(suf)] + x for x in sufs]
        return None

    def _unit_of(self, name):
        """Layers whose LoRA operand copies are laid out kind-major next to each other: the shared-input
        group of `name`, widened to ALL cross-attention k / v layers (they run as context chunks)."""
        if name.endswith((".attn2.to_k", ".attn2.to_v")):
            return self._ctx_names
        return self._group_of(name)

    def _stacked(self, layers, kind, rows, cols):
        """The `kind` ("a_fwd", "sb_fwd", "sb_t") operand copies of `layers`, laid out kind-major next to
        each other in lora_opnd, as ONE [rows, cols] view."""
        o = getattr(layers[0].lora, "o_" + kind)
        v = self.lora_opnd[o:o + rows * cols].view(rows, cols)
        last = getattr(layers[-1].lora, kind)
        assert last.data_ptr() == v.view(-1)[-last.numel():].data_ptr()
        return v

    def _build_groups(self, need_backward):
        """Stack the frozen weights (and view the kind-major LoRA operand copies) of every shared-input
        group so that q/k/v (resp. cross-attention k/v) run as ONE GEMM with N = g*C."""
        self.groups = {}
        for name in list(self.layers):
            for lead, _ in self._GROUPS:
                if not name.endswith(lead):
                    continue
                names = self._group_of(name)
                Ls = [self.layers[n] for n in names]
                assert all(L.bias is None and L.cin == Ls[0].cin and L.cout == Ls[0].cout for L in Ls)
                G = types.SimpleNamespace(names=names, layers=Ls, g=len(Ls), cin=Ls[0].cin, cout=Ls[0].cout)
                G.w_stack = torch.cat([L.w_fwd for L in Ls], 0).contiguous()
                G.w_t_cat = None
                if all(L.w_t is not None for L in Ls):
                    G.w_t_cat = torch.cat([L.w_t for L in Ls], 1).contiguous()   # [cin, g*C]
                for i, L in enumerate(Ls):
                    L.w_fwd = G.w_stack[i * G.cout:(i + 1) * G.cout]
                    L.w_t = None
                G.lora = all(L.lora is not None for L in Ls)
                if G.lora:
                    r, g = self.r, G.g
                    G.a_stack = self._stacked(Ls, "a_fwd", g * r, G.cin)
                    G.sb_stack = self._stacked(Ls, "sb_fwd", g * G.cout, r)
                    G.sbt_stack = self._stacked(Ls, "sb_t", g * r, G.cout)
                self.groups[name] = G

    def _build_temb_group(self):
        """Stacked operands of the time-embedding projections: W [sum C_i, temb], bias [sum C_i] and
        the kind-major LoRA copies A [g*r, temb], s*B [sum C_i, r]."""
        Ls = [self.layers[n] for n in self._temb_names]
        G = types.SimpleNamespace(names=self._temb_names, layers=Ls, g=len(Ls), cin=Ls[0].cin)
        assert all(L.cin == G.cin and L.bias is not None for L in Ls)
        G.offs = [0]
        for L in Ls:
            G.offs.append(G.offs[-1] + L.cout)
        G.n_total = G.offs[-1]
        assert G.n_total < 65536
        G.bn = 160 if all(o % 160 == 0 for o in G.offs) else 64
        G.index = {n: i for i, n in enumerate(G.names)}
        G.w_stack = torch.cat([L.w_fwd for L in Ls], 0).contiguous()
        G.bias = torch.cat([L.bias for L in Ls]).contiguous()
        for i, L in enumerate(Ls):
            L.w_fwd = G.w_stack[G.offs[i]:G.offs[i + 1]]
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

    def temb_all(self, st, lora):
        """All time_emb_proj layers of one pass: out[B, sum C_i] = [st | T] @ [W ; N-ranged s*B_i]^T + b.
        Returns (out, T): resnet i uses the column view out[:, offs[i]:offs[i+1]] as its row vector and
        column block i of T for its LoRA weight gradients."""
        G, r = self.temb_group, self.r
        T = self._lora_down(st[:self._lrows(st.shape[0])], G.a_stack) if lora and G.lora else None
        out = self._stacked_gemm(st, G.w_stack, T, getattr(G, "sb_stack", None),
                                 [(i * r, G.offs[i], G.offs[i + 1]) for i in range(G.g)], G.n_total,
                                 block_n=G.bn, bias=G.bias)
        return out, T

    def _build_ctx_group(self):
        """Cross-attention k / v of ALL transformer blocks from the text context (they depend on nothing
        else): A copies of every layer stacked [n_layers*r, ctx_dim] for ONE down-projection GEMM, and the
        frozen weights + s*B copies stacked per chunk (blocks of one width, at most 11 blocks = 22 N-ranged
        LoRA entries + the base entry <= PCM_MAX_PROG)."""
        self.ctx_group = None
        if not self._ctx_names:
            return
        names = self._ctx_names
        Ls = [self.layers[n] for n in names]
        assert all(L.bias is None and L.cin == Ls[0].cin for L in Ls) and len(names) % 2 == 0
        CG = types.SimpleNamespace(names=names, cin=Ls[0].cin, nl=len(names), chunks=[], where={})
        CG.lora = all(L.lora is not None for L in Ls)
        if CG.lora:
            CG.a_stack = self._stacked(Ls, "a_fwd", CG.nl * self.r, CG.cin)
        cur = None
        for b in range(len(names) // 2):
            lead = names[2 * b]
            assert lead.endswith(".attn2.to_k") and names[2 * b + 1] == lead[:-1] + "v"
            G = self.groups[lead]
            if cur is None or cur.cout != G.cout or len(cur.blocks) == 11:
                cur = types.SimpleNamespace(cout=G.cout, blocks=[], first=2 * b)
                CG.chunks.append(cur)
            CG.where[lead[:-len(".attn2.to_k")]] = (len(CG.chunks) - 1, len(cur.blocks))
            cur.blocks.append(G)
        for ch in CG.chunks:
            ch.n_total = 2 * ch.cout * len(ch.blocks)
            assert ch.n_total < 65536
            ch.bn = 160 if ch.cout % 160 == 0 else 64
            ch.w_stack = torch.cat([G.w_stack for G in ch.blocks], 0).contiguous()
            if CG.lora:
                ch.sb_stack = self._stacked([L for G in ch.blocks for L in G.layers], "sb_fwd", ch.n_total, self.r)
        self.ctx_group = CG

    def ctx_kv_all(self, ctx, lora):
        """{transformer block: (k, v, T)} for one pass: k / v are column views [M, C] of the chunk outputs,
        T the block's two columns blocks [Ml, 2r] of the stacked LoRA down-projection (None without LoRA)."""
        CG, r = self.ctx_group, self.r
        T = self._lora_down(ctx[:self._lrows(ctx.shape[0])], CG.a_stack) if lora and CG.lora else None
        outs = [self._stacked_gemm(ctx, ch.w_stack, T, getattr(ch, "sb_stack", None),
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

    def _block_weights(self):
        """Store every frozen GEMM weight K-blocked ([K/64][N][64], pcm_bsrc.kblocked): the operand tile of
        a K block becomes one contiguous run in HBM.  Matters for the small-M layers (8x8 / 16x16 levels,
        target pass), which stream their weights once per launch: a row-major tile is N separate
        128-byte segments K*2 bytes apart."""
        members = set()
        for G in list(self.groups.values()) + [self.temb_group]:
            members.update(id(L) for L in G.layers)
            G.w_stack = ops.kblock(G.w_stack)
            if getattr(G, "w_t_cat", None) is not None:
                G.w_t_cat = ops.kblock(G.w_t_cat)
        if self.ctx_group is not None:
            for ch in self.ctx_group.chunks:
                ch.w_stack = ops.kblock(ch.w_stack)
        for L in self.layers.values():
            if id(L) in members:
                L.w_fwd = None          # only reachable through the group's stacked operand
                continue
            if L.w_fwd is not None and L.w_fwd.dim() == 2:
                L.w_fwd = ops.kblock(L.w_fwd)
            if L.w_t is not None and L.w_t.dim() == 2:
                L.w_t = ops.kblock(L.w_t)

    class _Side:
        """Run the enclosed launches on the wgrad side stream, ordered after everything enqueued so far
        on the current stream; `keep` tensors stay referenced until backward() joins the streams."""

        def __init__(self, net, keep):
            self.net, self.keep, self.ctx = net, keep, None

        def __enter__(self):
            n = self.net
            if not n.use_wstream:
                return self
            ev = torch.cuda.Event()
            ev.record()
            n.wstream.wait_event(ev)
            n._keep.extend(self.keep)
            self.ctx = torch.cuda.stream(n.wstream)
            self.ctx.__enter__()
            return self

        def __exit__(self, *a):
            if self.ctx is not None:
                self.ctx.__exit__(*a)
            return False

    def _join_side(self):
        if self.use_wstream:
            torch.cuda.current_stream().wait_stream(self.wstream)
            self._keep.clear()

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
        backward, no LoRA operands, no tape.  Every K-blocked operand that holds a LoRA target's frozen
        weight (single layers, the q/k/v stacks, the time_emb_proj stack, the cross-attention k / v
        context chunks) gets a fused copy in ONE new bf16 buffer; every other tensor (norms, biases,
        conv_in / conv_out, time embedding) is this network's own.  Returns (net, fuse_table, fuse_work):
        fuse_table is the int64 [entries, 8] table of pcm_lora_fuse (ops.lora_fuse), one row per LoRA
        layer: {a_off, b_off, src, dst, n0 | N_total << 32, K | r << 32, n, work_begin}."""
        if not self.has_lora:
            raise ValueError("fused_inference_net needs a network built with lora=True")
        net = object.__new__(UNetB200)
        net.__dict__.update(self.__dict__)
        for k in ("lora_master", "lora_grad", "lora_opnd", "refresh_table", "refresh_work"):
            net.__dict__.pop(k, None)
        net.has_lora, net.use_wstream, net.wstream = False, False, None
        net.gradient_checkpointing = False
        net.lora_layers, net._keep, net._dkv_chunks = [], [], {}
        net.saved = net._temb = net._ctxkv = net.last_ctx_kv = None
        net._lb, net._plan_b = (1, 1), None
        # stacked operands: (source, [(layer, first row)]) of every operand holding a LoRA target
        stacks = []
        for L in self.lora_layers:
            if L.w_fwd is not None:     # not a member of a group: its own operand
                stacks.append(("layer", L.name, L.w_fwd, [(L, 0)]))
        for lead, G in self.groups.items():
            if lead.endswith(".attn1.to_q"):
                stacks.append(("group", lead, G.w_stack, [(L, i * G.cout) for i, L in enumerate(G.layers)]))
        TG = self.temb_group
        stacks.append(("temb", None, TG.w_stack, [(L, TG.offs[i]) for i, L in enumerate(TG.layers)]))
        if self.ctx_group is not None:
            for c, ch in enumerate(self.ctx_group.chunks):
                Ls = [L for G in ch.blocks for L in G.layers]
                stacks.append(("chunk", c, ch.w_stack, [(L, i * ch.cout) for i, L in enumerate(Ls)]))
        total = sum(src.numel() for _, _, src, _ in stacks)
        net.fused_weights = torch.empty(total, device=self.dev, dtype=BF16)
        rows, work, off, fused = [], 0, 0, {}
        for kind, key, src, members in stacks:
            dst = net.fused_weights[off:off + src.numel()].view(src.shape)
            off += src.numel()
            fused[(kind, key)] = dst
            K, ntot = src.shape[0] * 64, src.shape[1]
            assert sum(L.cout for L, _ in members) == ntot     # every row of the operand is a LoRA layer's
            for L, n0 in members:
                taps = L.k * L.k if L.kind == "conv" else 1
                assert L.lora is not None and taps * L.cin == K and L.cout % 64 == 0
                rows.append([L.lora.a_off, L.lora.b_off, src.data_ptr(), dst.data_ptr(), n0 | (ntot << 32),
                             K | (self.r << 32), L.cout, work])
                work += (L.cout // 64) * (K // 64)
        net.layers = {}
        for name, L in self.layers.items():
            C2 = _Layer()
            for s in _Layer.__slots__:
                setattr(C2, s, getattr(L, s))
            C2.lora, C2.w_t = None, None
            if ("layer", name) in fused:
                C2.w_fwd = fused[("layer", name)]
            net.layers[name] = C2
        net.groups = {}
        for lead, G in self.groups.items():
            if not lead.endswith(".attn1.to_q"):
                continue        # cross-attention k / v run as context chunks
            G2 = types.SimpleNamespace(**vars(G))
            G2.layers = [net.layers[n] for n in G.names]
            G2.w_stack, G2.w_t_cat, G2.lora = fused[("group", lead)], None, False
            net.groups[lead] = G2
        T2 = types.SimpleNamespace(**vars(TG))
        T2.layers = [net.layers[n] for n in TG.names]
        T2.w_stack, T2.lora = fused[("temb", None)], False
        net.temb_group = T2
        if self.ctx_group is not None:
            CG2 = types.SimpleNamespace(**vars(self.ctx_group))
            CG2.lora, CG2.chunks = False, []
            for c, ch in enumerate(self.ctx_group.chunks):
                ch2 = types.SimpleNamespace(**vars(ch))
                ch2.w_stack = fused[("chunk", c)]
                CG2.chunks.append(ch2)
            net.ctx_group = CG2
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

    def _conv_prog(self, xs, k, stride, cin_total):
        """(a_srcs, prog) of a k x k convolution over channel-concatenated sources xs."""
        if stride == 2:
            x = xs[0]
            planes = [x[:, p::2, q::2, :] for p in range(2) for q in range(2)]
            srcs = [ops.asrc_nhwc(pl) for pl in planes]
            prog = []
            for kh in range(3):
                for kw in range(3):
                    p, dh = _S2[kh]
                    q, dw = _S2[kw]
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

    def _merged_tiling(self, M, N, prog):
        """Tiling keywords of a block's main GEMM.  Empty (ops.gemm picks from M) except while backward()
        rebuilds a checkpointed block: then the (block_n, ksplit) the merged pass picked for its larger M,
        since pick_tiling splits K by M and the split decides how the fp32 sums round.  The LoRA
        down-projections already ran on the student rows alone and need nothing."""
        if self._plan_b is None:
            return {}
        bn, ks = ops.pick_tiling(M * self._plan_b // self._lb[1], N, sum(e[4] for e in prog))
        return dict(block_n=bn, ksplit=ks)

    def conv3(self, name, xs, lora, stride=1, rowvec=None, residual=None, out_fp32=False, save=None):
        """3x3 pad-1 convolution (+LoRA) over NHWC sources xs (channel concat), fused epilogue; appends its
        ConvRec to the list `save`."""
        L = self.layers[name]
        B, H, W, _ = xs[0].shape
        Ho, Wo = H // stride, W // stride
        M, N = B * Ho * Wo, L.cout
        srcs, prog = self._conv_prog(xs, 3, stride, L.cin)
        bs = [ops.bsrc(L.w_fwd)]
        T = None
        lbn = self._lrows(B)   # samples that carry the LoRA adapter (the leading ones of the batch)
        xl = xs if lbn == B else [x[:lbn] for x in xs]
        if lora and L.lora is not None:
            # T = A(x) only for the LoRA samples; the other samples see T rows that TMA zero-fills
            T = self._new(lbn, Ho, Wo, self.r)
            srcs_l, prog_l = (srcs, prog) if lbn == B else self._conv_prog(xl, 3, stride, L.cin)
            ops.gemm(srcs_l, [ops.bsrc(L.lora.a_fwd)], prog_l, lin=False, M=lbn * Ho * Wo, N=self.r,
                     geo=(Wo, Ho), out=T.view(lbn * Ho * Wo, self.r))
            prog = prog + [(len(srcs), 1, 0, 0, self.rc, 0, 0)]
            srcs = srcs + [ops.asrc_nhwc(T)]
            bs.append(ops.bsrc(L.lora.sb_fwd))
        out = self._new(B, Ho, Wo, N, dtype=torch.float32 if out_fp32 else BF16)
        ops.gemm(srcs, bs, prog, lin=False, M=M, N=N, geo=(Wo, Ho), out=out.view(M, N), bias=L.bias,
                 rowvec=rowvec, residual=None if residual is None else residual.reshape(M, N),
                 round_bf16=out_fp32, dep_a_src=None if T is None else len(srcs) - 1,
                 **self._merged_tiling(M, N, prog))
        if save is not None:
            save.append(ConvRec("conv3", name, xl, T, stride))
        return out

    def linear(self, name, xs, lora, residual=None, act=0, save=None):
        """nn.Linear / 1x1 conv over [M, C] matrices xs (channel concat) (+LoRA), fused epilogue; appends its
        LinearRec to the list `save`."""
        L = self.layers[name]
        M, N = xs[0].shape[0], L.cout
        srcs = [ops.asrc_mat(x) for x in xs]
        prog, coff = [], 0
        for si, x in enumerate(xs):
            prog.append((si, 0, 0, 0, x.shape[1] // 64, 0, coff))
            coff += x.shape[1]
        bs = [ops.bsrc(L.w_fwd)]
        T = None
        Ml = self._lrows(M)
        xl = xs if Ml == M else [x[:Ml] for x in xs]
        if lora and L.lora is not None:
            T = self._new(Ml, self.r)
            srcs_l = srcs if Ml == M else [ops.asrc_mat(x) for x in xl]
            ops.gemm(srcs_l, [ops.bsrc(L.lora.a_fwd)], prog, lin=True, M=Ml, N=self.r, out=T)
            prog = prog + [(len(srcs), 1, 0, 0, self.rc, 0, 0)]
            srcs = srcs + [ops.asrc_mat(T)]   # Ml rows: tiles past them read zeros (TMA bounds)
            bs.append(ops.bsrc(L.lora.sb_fwd))
        out = self._new(M, N)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=N, out=out, bias=L.bias, residual=residual, act=act,
                 dep_a_src=None if T is None else len(srcs) - 1, **self._merged_tiling(M, N, prog))
        if save is not None:
            save.append(LinearRec("linear", name, xl, T))
        return out

    def linear_group(self, lead, x, lora, save=None):
        """The g Linear layers of a shared-input group (attn1 q/k/v, attn2 k/v) as ONE GEMM:
        out[M, g*C] = x @ [W_0; ...; W_g-1]^T, layer i's LoRA up-projection entering as a K block that
        only feeds its own C output columns.  Returns the g column views of out; appends its GroupRec to
        the list `save`."""
        G, r = self.groups[lead], self.r
        g, Cc = G.g, G.cout
        xl = x[:self._lrows(x.shape[0])]
        T = self._lora_down(xl, G.a_stack) if lora and G.lora else None
        out = self._stacked_gemm(x, G.w_stack, T, getattr(G, "sb_stack", None),
                                 [(i * r, i * Cc, (i + 1) * Cc) for i in range(g)], g * Cc,
                                 block_n=160 if Cc % 160 == 0 else 64, dep_a_src=None if T is None else 1)
        if save is not None:
            save.append(GroupRec("lgroup", lead, xl, T))
        return [out[:, i * Cc:(i + 1) * Cc] for i in range(g)]

    def gn(self, name, xs, B, HW, eps, silu, save=None):
        L = self.layers[name]
        C = sum(x.shape[-1] for x in xs)
        out = self._new(B * HW, C)
        stats = self._new(B, self.cfg.norm_num_groups, 2, dtype=torch.float32)
        x2 = xs[1] if len(xs) > 1 else None
        if self._plan_b is None:
            ops.groupnorm_fwd(xs[0], x2, L.gamma, L.beta, eps, silu, out, stats, B, HW, self.cfg.norm_num_groups)
        else:   # a rebuilt block: merge each image's statistics from the merged pass's partition
            ops.groupnorm_fwd_part(xs[0], x2, L.gamma, L.beta, eps, silu, out, stats, B, self._plan_b, HW,
                                   self.cfg.norm_num_groups)
        if save is not None:
            lb = self._lrows(B)
            save.append(GNRec("gn", name, xs if lb == B else [x[:lb * HW] for x in xs], stats[:lb], eps, silu, lb, HW))
        return out

    def ln(self, name, x, save=None):
        L = self.layers[name]
        out = torch.empty_like(x)
        stats = self._new(x.shape[0], 2, dtype=torch.float32)
        ops.layernorm_fwd(x, L.gamma, L.beta, out, stats)
        if save is not None:
            Ml = self._lrows(x.shape[0])
            save.append(LNRec("ln", name, x[:Ml], stats[:Ml]))
        return out

    def attention(self, q, k, v, B, Sq, Skv, heads, save=None):
        D = q.shape[1] // heads
        out = self._new(q.shape[0], q.shape[1])
        lse = self._new(B, heads, Sq, dtype=torch.float32)
        ops.attn_fwd(q, k, v, out, lse, B, heads, Sq, Skv, D, D ** -0.5)
        if save is not None:
            lb = self._lrows(B)
            save.append(AttnRec("attn", q[:lb * Sq], k[:lb * Skv], v[:lb * Skv], out[:lb * Sq], lse[:lb], lb, Sq, Skv,
                                heads))
        return out

    # ------------------------------------------------------------------------------------
    # blocks (forward): each returns (out, block record)
    # ------------------------------------------------------------------------------------
    def resnet(self, p, xs, st, lora, save):
        """xs: list of NHWC sources (skip concat = 2 sources).  Returns ([B,H,W,Cout], ResnetRec)."""
        B, H, W, _ = xs[0].shape
        HW = H * W
        cin = sum(x.shape[-1] for x in xs)
        cout = self.layers[p + ".conv1"].cout
        flat = [x.view(B * HW, x.shape[-1]) for x in xs]
        s = [] if save else None        # this block's op records
        h = self.gn(p + ".norm1", flat, B, HW, 1e-5, True, s)
        norm1 = _last(s)
        G = self.temb_group
        i = G.index[p + ".time_emb_proj"]
        out_all, T_all = self._temb
        # the grouped launch of temb_all computed this layer: its record only names the column block
        temb = TembRec("linear", p + ".time_emb_proj", [st[:self._lrows(st.shape[0])]], T_all, i * self.r)
        h = self.conv3(p + ".conv1", [h.view(B, H, W, cin)], lora, rowvec=out_all[:, G.offs[i]:G.offs[i + 1]],
                       save=s)
        conv1 = _last(s)
        h = self.gn(p + ".norm2", [h.view(B * HW, cout)], B, HW, 1e-5, True, s)
        norm2 = _last(s)
        sc, shortcut = xs[0], None
        if cin != cout:
            sc = self.linear(p + ".conv_shortcut", flat, lora, save=s).view(B, H, W, cout)
            shortcut = _last(s)
        out = self.conv3(p + ".conv2", [h.view(B, H, W, cout)], lora, residual=sc, save=s)
        return out, ResnetRec(p, norm1, temb, conv1, norm2, shortcut, _last(s), takes_skip=len(xs) == 2)

    def _level_of(self, name):
        """Resolution level of a block name (selects transformer depth and head count)."""
        nb = len(self.cfg.block_out_channels)
        parts = name.split(".")
        if parts[0] == "mid_block":
            return nb - 1
        i = int(parts[1])
        return i if parts[0] == "down_blocks" else nb - 1 - i

    def transformer(self, p, x, ctx, lora, save):
        """Transformer2DModel: GN -> proj_in -> depth x BasicTransformerBlock -> proj_out -> + residual.
        proj_in / proj_out are 1x1 convolutions (SD1.5) or nn.Linear (SDXL, use_linear_projection):
        on NHWC tokens both are the same GEMM."""
        B, H, W, C = x.shape
        S, M = H * W, B * H * W
        level = self._level_of(p)
        heads = self.cfg.heads(level)
        xf = x.view(M, C)
        s = [] if save else None        # this block's op records
        g = self.gn(p + ".norm", [xf], B, S, 1e-6, False, s)
        norm = _last(s)
        h = self.linear(p + ".proj_in", [g], lora, save=s)
        proj_in = _last(s)
        blocks = []
        for d in range(self.cfg.depth(level)):
            t = p + f".transformer_blocks.{d}"
            b = [] if save else None    # the op records of one transformer block, in TBlockRec order
            n = self.ln(t + ".norm1", h, b)
            q, k, v = self.linear_group(t + ".attn1.to_q", n, lora, save=b)
            a = self.attention(q, k, v, B, S, S, heads, b)
            h = self.linear(t + ".attn1.to_out.0", [a], lora, residual=h, save=b)
            n = self.ln(t + ".norm2", h, b)
            q = self.linear(t + ".attn2.to_q", [n], lora, save=b)
            k, v, Tkv = self._ctxkv[t]
            if save:    # k / v came from the context chunks of ctx_kv_all; Tkv is this block's window of T
                b.append(GroupRec("lgroup", t + ".attn2.to_k", ctx[:self._lrows(ctx.shape[0])], Tkv))
            a = self.attention(q, k, v, B, S, ctx.shape[0] // B, heads, b)
            h = self.linear(t + ".attn2.to_out.0", [a], lora, residual=h, save=b)
            n = self.ln(t + ".norm3", h, b)
            u = self.linear(t + ".ff.net.0.proj", [n], lora, save=b)
            gg = self._new(M, u.shape[1] // 2)
            ops.geglu_fwd(u, gg)
            if save:
                b.append(GegluRec("geglu", u[:self._lrows(M)]))
            h = self.linear(t + ".ff.net.2", [gg], lora, residual=h, save=b)
            blocks.append(TBlockRec._make(b) if save else None)
        out = self.linear(p + ".proj_out", [h], lora, residual=xf, save=s)
        return out.view(B, H, W, C), TransformerRec(p, norm, proj_in, blocks, _last(s))

    def resample(self, name, x, lora, save, up):
        """Downsampler (stride-2 convolution) or upsampler (nearest 2x, then the convolution)."""
        s = [] if save else None
        if not up:
            out = self.conv3(name, [x], lora, stride=2, save=s)
        else:
            B, H, W, C = x.shape
            xu = self._new(B, 2 * H, 2 * W, C)
            ops.upsample2x_fwd(x, xu)
            out = self.conv3(name, [xu], lora, save=s)
        return out, ResampleRec(name, _last(s), up)

    def _block(self, kind, name, xs, st, ctx, lora, save, up=False):
        """One block's forward: (out, record)."""
        if kind == "resnet":
            return self.resnet(name, xs, st, lora, save)
        if kind == "transformer":
            return self.transformer(name, xs[0], ctx, lora, save)
        return self.resample(name, xs[0], lora, save, up)

    def _lrows(self, n):
        """Rows / samples of an n-row (batch-major) tensor that belong to the LoRA samples."""
        lb, bt = self._lb
        return n * lb // bt

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
        tensor are freed as the forward proceeds.  The time-embedding and context projections of the pass
        stay referenced (small), and the head's GroupNorm record keeps a copy of its student rows.
        backward() then rebuilds one block's full record at a time."""
        cfg = self.cfg
        lora = lora and self.has_lora
        B, H, W, _ = sample.shape
        self._lb = (lora_batch if (lora and lora_batch) else B, B)
        c0 = cfg.block_out_channels[0]
        emb = self._new(B, c0)
        ops.timestep_embed(timesteps, emb)
        hemb = self.linear("time_embedding.linear_1", [emb], False, act=1)
        if not cfg.addition_embed:
            st = self.linear("time_embedding.linear_2", [hemb], False, act=1)  # silu(temb)
        else:
            # "text_time": emb = time_embedding(t) + add_embedding(cat[text_embeds, sinusoid(time_ids)]);
            # every consumer takes silu(emb): the sum and the SiLU run in the last GEMM's epilogue
            if added_cond is None:
                raise ValueError("this UNet needs added_cond = (text_embeds, time_ids) (addition_embed_type text_time)")
            text_embeds, time_ids = added_cond
            temb = self.linear("time_embedding.linear_2", [hemb], False)
            tid = self._new(B * cfg.num_time_ids, cfg.addition_time_embed_dim)
            ops.timestep_embed(time_ids.reshape(-1), tid)
            add_in = torch.cat([text_embeds.to(BF16), tid.view(B, -1)], dim=1).contiguous()  # [B, 2816] glue
            ah = self.linear("add_embedding.linear_1", [add_in], False, act=1)
            st = self.linear("add_embedding.linear_2", [ah], False, residual=temb, act=1)
        self._temb = self.temb_all(st, lora)
        # cross-attention k / v of every block: given (ctx_kv: another pass of this step already projected
        # the same context with the same weights) or computed here in a few grouped GEMMs
        if ctx_kv is not None:
            assert not save
            self._ctxkv = ctx_kv
        else:
            self._ctxkv = self.ctx_kv_all(ctx, lora) if self.ctx_group is not None else None
        self.last_ctx_kv = self._ctxkv if lora else None
        x = self._new(B, H, W, c0)
        Lci = self.layers["conv_in"]
        ops.conv3x3_c4(sample, Lci.w_c4, Lci.bias, x, sgn=1, round_in=True)
        tape, skips = [], [x]       # tape: the block records in forward order
        ck = save and self.gradient_checkpointing
        lb = self._lb[0]
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
                return self._block(kind, name, xs, st, ctx, lora, False, up)[0]
            out, rec = self._block(kind, name, xs, st, ctx, lora, save, up)
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
        g = self.gn("conv_norm_out", [x.view(Bx * Hx * Wx, Cx)], Bx, Hx * Wx, 1e-5, True, head)
        eps = self.conv3("conv_out", [g.view(Bx, Hx, Wx, Cx)], False, out_fp32=True)
        if save:
            rebuild = None
            if ck:
                h = head[0]      # already the student rows: views of the merged pass's last activation
                if lb != B:
                    head[0] = h._replace(xs=[t.clone() for t in h.xs], stats=h.stats.clone())
                rebuild = self._rebuild_state(lora, B, st, ctx)
            self.saved = (tape, head[0], (lb, H, W), rebuild)
        return eps

    def _rebuild_state(self, lora, B, st, ctx):
        """What rebuilding a checkpointed block of this pass needs besides its inputs: the student rows of
        the pass's time embedding, of its grouped time_emb_proj output and of its context k / v."""
        lb = self._lb[0]
        out_all, T = self._temb
        kv = self._ctxkv
        S = ctx.shape[0] // B
        if kv is not None:
            kv = {t: (k[:lb * S], v[:lb * S], Tkv) for t, (k, v, Tkv) in kv.items()}
        return types.SimpleNamespace(lora=lora, B=B, lb=lb, st=st[:lb], ctx=ctx[:lb * S], temb=(out_all[:lb], T),
                                     ctxkv=kv)

    def _rebuild(self, ck, state):
        """The full record of a checkpointed block: its forward once more, on the saved student rows, with
        the launch plans of the merged pass that first ran it, so that every tensor of the record is
        bitwise the one the stored tape would hold."""
        prev = self._lb, self._temb, self._ctxkv
        self._lb, self._temb, self._ctxkv = (state.lb, state.lb), state.temb, state.ctxkv
        self._plan_b = state.B if state.B != state.lb else None
        try:
            return self._block(ck.kind, ck.name, ck.xs, state.st, state.ctx, state.lora, True, ck.up)[1]
        finally:
            self._lb, self._temb, self._ctxkv = prev
            self._plan_b = None

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

    def linear_bwd(self, rec, dy, need_dx=True, t_c0=0):
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
            with UNetB200._Side(self, (dy, rec.T, dt, *rec.xs)):
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

    def linear_group_bwd(self, rec, dpk, need_dx=True):
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
            with UNetB200._Side(self, (dpk, T, dT, x)):
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

    def conv3_bwd(self, rec, dy, need_dx=True):
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
            with UNetB200._Side(self, (dy, rec.T, dt, rec.xs)):
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

    def attn_bwd(self, rec, dout):
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
            if key not in self._dkv_chunks:
                self._dkv_chunks[key] = self._new(k.shape[0], ld)
            pk = self._dkv_chunks[key][:, col0:col0 + 2 * Cc]
            dk, dv = pk[:, :Cc], pk[:, Cc:]
        delta = torch.empty_like(rec.lse)
        ops.attn_bwd(q, k, v, rec.out, dout, rec.lse, delta, dq, dk, dv, rec.B, Hh, rec.Sq, rec.Skv, D, D ** -0.5)
        return dq, pk

    # ------------------------------------------------------------------------------------
    # block backward
    # ------------------------------------------------------------------------------------
    def resnet_bwd(self, blk, dout, need_dx=True):
        """dout [B,H,W,Cout].  Returns the gradients (NHWC) of the input and of the skip source (None
        without a skip), or (None, None) without need_dx."""
        B, H, W, cout = dout.shape
        M = B * H * W
        dh2 = self.conv3_bwd(blk.conv2, dout)                          # grad wrt silu(gn2(h1))
        # grad wrt h1 [M, cout]; its per-image column sums (= d tproj[b, n], the time-embedding
        # branch) are accumulated by the same kernel
        cs32 = self._new(B, cout, dtype=torch.float32)
        dh1, _ = self.gn_bwd(blk.norm2, dh2.view(M, cout), colsum=cs32)
        # the time-embedding branch ends in LoRA weight gradients only: all of it on the side stream
        with UNetB200._Side(self, (cs32,)):
            drow = self._new(B, cout)
            ops.cast_f32_bf16(cs32, drow)
            self._keep.append(drow)
            self.linear_bwd(blk.temb, drow, need_dx=False, t_c0=blk.temb.t_c0)
        dh = self.conv3_bwd(blk.conv1, dh1.view(B, H, W, cout), need_dx=need_dx)
        dsc = dout.view(M, cout)
        if blk.shortcut is not None:
            dsc = self.linear_bwd(blk.shortcut, dsc, need_dx=need_dx)
        if not need_dx:
            return None, None
        dx1, dx2 = self.gn_bwd(blk.norm1, dh.view(M, -1), add=dsc)
        return dx1.view(B, H, W, -1), None if dx2 is None else dx2.view(B, H, W, -1)

    def transformer_bwd(self, blk, dout):
        """dout [B,H,W,C]; returns dx [B,H,W,C]."""
        B, H, W, C = dout.shape
        M = B * H * W
        do = dout.view(M, C)
        dh = self.linear_bwd(blk.proj_out, do)
        for b in reversed(blk.blocks):
            dh3 = dh
            dgg = self.linear_bwd(b.ff_out, dh3)
            du = torch.empty_like(b.geglu.u)
            ops.geglu_bwd(dgg, b.geglu.u, du)
            dn3 = self.linear_bwd(b.ff_in, du)
            dh2 = self.ln_bwd(b.norm3, dn3, add=dh3)
            da2 = self.linear_bwd(b.attn2_out, dh2)
            dq2, dkv2 = self.attn_bwd(b.attn2, da2)
            with UNetB200._Side(self, (dkv2,)):     # feeds weight gradients only: off the dgrad chain
                self.linear_group_bwd(b.attn2_kv, dkv2, need_dx=False)
            dn2 = self.linear_bwd(b.attn2_q, dq2)
            dh1 = self.ln_bwd(b.norm2, dn2, add=dh2)
            da1 = self.linear_bwd(b.attn1_out, dh1)
            _, dqkv = self.attn_bwd(b.attn1, da1)
            dn1 = self.linear_group_bwd(b.attn1_qkv, dqkv)
            dh = self.ln_bwd(b.norm1, dn1, add=dh1)
        dg = self.linear_bwd(blk.proj_in, dh)
        dx, _ = self.gn_bwd(blk.norm, dg, add=do)
        return dx.view(B, H, W, C)

    def resample_bwd(self, blk, dout):
        dx = self.conv3_bwd(blk.conv, dout)
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
        self._dkv_chunks = {}
        boffs = self.block_grad_offsets() if grad_ready is not None else None
        Lco = self.layers["conv_out"]
        c0 = Lco.cin
        dg = self._new(B, H, W, c0)
        ops.conv3x3_c4(d_eps, Lco.w_c4_t, None, dg, sgn=-1, round_in=False)
        d, _ = self.gn_bwd(head, dg.view(B * H * W, c0))
        d = d.view(B, H, W, c0)
        dskips = []     # gradients of the up path's skip inputs; the last one left (conv_in's output) is unused
        done = None     # the block walked before the current one
        side = []       # checkpointing: (event, tensors) of the weight-gradient work of the last blocks walked
        for i in reversed(range(len(tape))):
            blk = tape[i]
            if blk.pushes_skip:
                d = ops.add_bf16(d, dskips.pop(), torch.empty_like(d))
            # the block walked before has been fully enqueued by now: its gradients are final once the
            # weight-gradient stream drains
            if grad_ready is not None and boffs.get(done) is not None:
                with UNetB200._Side(self, ()):
                    grad_ready(boffs[done])
            if isinstance(blk, CheckpointRec):
                tape[i] = None              # the rebuilt record holds what the backward still reads
                blk = self._rebuild(blk, rebuild)
            if isinstance(blk, ResnetRec):
                d, dskip = self.resnet_bwd(blk, d, need_dx=i > 0)
                if blk.takes_skip:
                    dskips.append(dskip)
            elif isinstance(blk, TransformerRec):
                d = self.transformer_bwd(blk, d)
            else:
                d = self.resample_bwd(blk, d)
            done = blk.name
            if rebuild is not None:
                self._release_side(side)
        if grad_ready is not None:
            with UNetB200._Side(self, ()):
                grad_ready(0)
        self._join_side()
        side.clear()
        self.saved = None

    def _release_side(self, side):
        """Checkpointing: the tensors the weight-gradient stream reads stay referenced (_Side keeps them)
        until that stream is done with them.  Joining the streams after every block would serialise the
        weight gradients with the backward chain, so release them one block late: the current stream
        waits for the side work of the block walked before this one, which has had a whole block's
        backward to finish, and then drops its tensors."""
        if not self.use_wstream:
            return
        ev = torch.cuda.Event()
        ev.record(self.wstream)
        side.append((ev, self._keep))
        self._keep = []
        if len(side) > 1:
            ev, _ = side.pop(0)
            torch.cuda.current_stream().wait_event(ev)
