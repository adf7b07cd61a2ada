"""H100 (sm_90a) SD1.5 UNet (student / target with fused LoRA, frozen teacher) -- host orchestration.

Python only sequences C-ABI kernel launches (pcm_b200.ops); every FLOP runs in libpcm_b200.so.
Mirrors the call `unet(sample, timestep, encoder_hidden_states=...).sample` of diffusers'
UNet2DConditionModel wrapped by peft (train_pcm_lora_sd15.py:1192-1198 student, :1219-1244
teacher, :1263-1268 target) and its autograd backward (:1296), with:
  * activations NHWC bf16, one rounding per materialised tensor (bf16 autocast semantics);
  * LoRA unmerged: T = A(x) as a 64-wide GEMM, then s*B*T enters the base GEMM as one extra
    64-wide K block (same wgmma accumulator), so `base(x) + B(A(x)) * scaling` is one kernel;
  * skip concats never materialised (two K segments / two GroupNorm sources);
  * backward = explicit tape: dgrad through every layer, wgrad for LoRA factors only.
Parameters use diffusers state-dict names; LoRA factors live in ONE flat fp32 buffer
(`lora_master`), their gradients in `lora_grad`.
"""
import types

import torch

from . import ops
from .config import UNetConfig, is_lora_target, layer_table

BF16 = torch.bfloat16
TAPS3 = ops.TAPS3
# stride-2 3x3 pad-1: kernel index -> (input parity, shift in the parity plane)
_S2 = ((1, -1), (0, 0), (1, 0))


class _Lora:
    __slots__ = ("a_off", "b_off", "a_fwd", "sb_fwd", "sb_t", "a_t", "gA", "gB", "opnd_off",
                 "o_a_fwd", "o_sb_fwd", "o_sb_t", "o_a_t")


class _Layer:
    __slots__ = ("name", "kind", "cin", "cout", "k", "w_fwd", "w_t", "bias", "gamma", "beta", "lora",
                 "w_c4", "w_c4_t")


class UNetB200:
    def __init__(self, cfg: UNetConfig, state_dict, device, need_backward=True, lora=True):
        self.cfg, self.dev = cfg, device
        self.r = cfg.lora_rank
        self.scale = cfg.lora_scale
        self.layers = {}
        self.has_lora = lora
        tab = layer_table(cfg)
        # every resnet's time_emb_proj reads the same silu(temb): one grouped GEMM per pass
        # (1 base K entry + one N-ranged LoRA entry per layer must fit the K program)
        self._temb_names = [n for n, *_ in tab if n.endswith(".time_emb_proj")]
        if not 2 <= len(self._temb_names) <= 23:
            self._temb_names = []
        # every cross-attention k / v projection reads the same text context: a few grouped GEMMs per
        # pass (chunks of <= 11 transformer blocks of one width, _build_ctx_group) instead of one per block
        import os as _os0
        self._ctx_names = [n for n, _, ci, *_ in tab if n.endswith((".attn2.to_k", ".attn2.to_v"))]
        _co = {n: co for n, _, _, co, _ in tab}
        self._ctx_names.sort(key=lambda n: _co[n])        # stable: blocks of one width become neighbours
        if (_os0.environ.get("PCM_CTX_GROUP", "1") == "0" or len(self._ctx_names) < 4 or
                len({ci for n, _, ci, *_ in tab if n in set(self._ctx_names)}) != 1):
            self._ctx_names = []
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
                assert self.r == 64 and L.cin % 64 == 0 and L.cout % 64 == 0
                work += (taps * L.cin) // 64 + L.cout // 64     # 64x64 tiles of A, then of B
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
        # LoRA weight-gradient GEMMs are off the dgrad critical path (they only feed the optimiser):
        # they run on a side stream and fill SMs the main backward chain leaves idle
        import os as _os
        self.use_wstream = (torch.device(device).type == "cuda" and need_backward and lora and
                            _os.environ.get("PCM_WGRAD_STREAM", "1") != "0")
        self.wstream = torch.cuda.Stream(device=device) if self.use_wstream else None
        self._keep = []

    _GROUPS = ((".attn1.to_q", (".attn1.to_q", ".attn1.to_k", ".attn1.to_v")),
               (".attn2.to_k", (".attn2.to_k", ".attn2.to_v")))

    def _group_of(self, name):
        """Names of the shared-input Linear group `name` belongs to (attn1 q/k/v, attn2 k/v, all
        time_emb_proj layers), or None."""
        if name.endswith(".time_emb_proj") and self._temb_names:
            return self._temb_names
        for _, sufs in self._GROUPS:
            for suf in sufs:
                if name.endswith(suf):
                    return [name[:-len(suf)] + x for x in sufs]
        return None

    def _unit_of(self, name):
        """Layers whose LoRA operand copies are laid out kind-major next to each other: the shared-input
        group of `name`, widened to ALL cross-attention k / v layers when they run as context chunks."""
        if self._ctx_names and name.endswith((".attn2.to_k", ".attn2.to_v")):
            return self._ctx_names
        return self._group_of(name)

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
                    lo0 = Ls[0].lora
                    op = self.lora_opnd
                    G.a_stack = op[lo0.o_a_fwd:lo0.o_a_fwd + g * r * G.cin].view(g * r, G.cin)
                    G.sb_stack = op[lo0.o_sb_fwd:lo0.o_sb_fwd + g * G.cout * r].view(g * G.cout, r)
                    G.sbt_stack = op[lo0.o_sb_t:lo0.o_sb_t + g * G.cout * r].view(g * r, G.cout)
                    assert Ls[-1].lora.a_fwd.data_ptr() == G.a_stack[(g - 1) * r:].data_ptr()
                    assert Ls[-1].lora.sb_fwd.data_ptr() == G.sb_stack[(g - 1) * G.cout:].data_ptr()
                    assert Ls[-1].lora.sb_t.data_ptr() == G.sbt_stack[(g - 1) * r:].data_ptr()
                self.groups[name] = G

    def _build_temb_group(self):
        """Stacked operands of the time-embedding projections: W [sum C_i, temb], bias [sum C_i] and
        the kind-major LoRA copies A [g*r, temb], s*B [sum C_i, r]."""
        self.temb_group = None
        if not self._temb_names:
            return
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
            r, g = self.r, G.g
            lo0, op = Ls[0].lora, self.lora_opnd
            G.a_stack = op[lo0.o_a_fwd:lo0.o_a_fwd + g * r * G.cin].view(g * r, G.cin)
            G.sb_stack = op[lo0.o_sb_fwd:lo0.o_sb_fwd + G.n_total * r].view(G.n_total, r)
            assert Ls[-1].lora.a_fwd.data_ptr() == G.a_stack[(g - 1) * r:].data_ptr()
            assert Ls[-1].lora.sb_fwd.data_ptr() == G.sb_stack[G.offs[-2]:].data_ptr()
        self.temb_group = G

    def temb_all(self, st, lora):
        """All time_emb_proj layers of one pass: out[B, sum C_i] = [st | T] @ [W ; N-ranged s*B_i]^T + b.
        Returns (out, T): resnet i uses the column view out[:, offs[i]:offs[i+1]] as its row vector and
        column block i of T for its LoRA weight gradients."""
        G = self.temb_group
        B = st.shape[0]
        Ml = self._lrows(B)
        srcs, bs = [ops.asrc_mat(st)], [ops.bsrc(G.w_stack)]
        prog = [(0, 0, 0, 0, G.cin // 64, 0, 0)]
        T = None
        if lora and G.lora:
            r = self.r
            T = self._new(Ml, G.g * r)
            ops.gemm([ops.asrc_mat(st[:Ml])], [ops.bsrc(G.a_stack)], prog, lin=True, M=Ml, N=G.g * r, out=T)
            srcs.append(ops.asrc_mat(T))
            bs.append(ops.bsrc(G.sb_stack))
            prog = prog + [(1, 1, 0, 0, 1, i * r, 0, G.offs[i], G.offs[i + 1]) for i in range(G.g)]
        out = self._new(B, G.n_total)
        ops.gemm(srcs, bs, prog, lin=True, M=B, N=G.n_total, out=out, bias=G.bias, block_n=G.bn)
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
        assert all(L.bias is None for L in Ls) and len(names) % 2 == 0
        CG = types.SimpleNamespace(names=names, cin=Ls[0].cin, nl=len(names), chunks=[], where={})
        CG.lora = all(L.lora is not None for L in Ls)
        if CG.lora:
            lo0, op = Ls[0].lora, self.lora_opnd
            CG.a_stack = op[lo0.o_a_fwd:lo0.o_a_fwd + CG.nl * self.r * CG.cin].view(CG.nl * self.r, CG.cin)
            assert Ls[-1].lora.a_fwd.data_ptr() == CG.a_stack[(CG.nl - 1) * self.r:].data_ptr()
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
                lo = self.layers[names[ch.first]].lora
                ch.sb_stack = self.lora_opnd[lo.o_sb_fwd:lo.o_sb_fwd + ch.n_total * self.r].view(ch.n_total, self.r)
                last = ch.blocks[-1].layers[-1].lora
                assert last.sb_fwd.data_ptr() == ch.sb_stack[ch.n_total - ch.cout:].data_ptr()
        self.ctx_group = CG

    def ctx_kv_all(self, ctx, lora):
        """{transformer block: (k, v, T)} for one pass: k / v are column views [M, C] of the chunk outputs,
        T the block's two columns blocks [Ml, 2r] of the stacked LoRA down-projection (None without LoRA)."""
        CG, r = self.ctx_group, self.r
        M = ctx.shape[0]
        Ml = self._lrows(M)
        base = [(0, 0, 0, 0, CG.cin // 64, 0, 0)]
        T = None
        if lora and CG.lora:
            T = self._new(Ml, CG.nl * r)
            ops.gemm([ops.asrc_mat(ctx[:Ml])], [ops.bsrc(CG.a_stack)], base, lin=True, M=Ml, N=CG.nl * r, out=T)
        outs = []
        for ch in CG.chunks:
            srcs, bs, prog = [ops.asrc_mat(ctx)], [ops.bsrc(ch.w_stack)], list(base)
            if T is not None:
                srcs.append(ops.asrc_mat(T))
                bs.append(ops.bsrc(ch.sb_stack))
                prog += [(1, 1, 0, 0, 1, (ch.first + i) * r, 0, i * ch.cout, (i + 1) * ch.cout)
                         for i in range(2 * len(ch.blocks))]
            out = self._new(M, ch.n_total)
            ops.gemm(srcs, bs, prog, lin=True, M=M, N=ch.n_total, out=out, block_n=ch.bn)
            outs.append(out)
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
        128-byte segments K*2 bytes apart.  PCM_KBLOCK=0 keeps the row-major layout."""
        import os as _os
        if _os.environ.get("PCM_KBLOCK", "1") == "0":
            return
        members = set()
        for G in list(self.groups.values()) + ([self.temb_group] if self.temb_group is not None else []):
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

    def conv3(self, name, xs, lora, stride=1, rowvec=None, residual=None, out_fp32=False, save=None):
        """3x3 pad-1 convolution (+LoRA) over NHWC sources xs (channel concat), fused epilogue."""
        L = self.layers[name]
        B, H, W, _ = xs[0].shape
        Ho, Wo = H // stride, W // stride
        M, N = B * Ho * Wo, L.cout
        srcs, prog = self._conv_prog(xs, 3, stride, L.cin)
        bs = [ops.bsrc(L.w_fwd)]
        T = None
        lbn = self._lrows(B)   # samples that carry the LoRA adapter (the leading ones of the batch)
        if lora and L.lora is not None:
            # T = A(x) only for the LoRA samples; the other samples see T rows that TMA zero-fills
            T = self._new(lbn, Ho, Wo, self.r)
            xl = xs if lbn == B else [x[:lbn] for x in xs]
            srcs_l, prog_l = (srcs, prog) if lbn == B else self._conv_prog(xl, 3, stride, L.cin)
            ops.gemm(srcs_l, [ops.bsrc(L.lora.a_fwd)], prog_l, lin=False, M=lbn * Ho * Wo, N=self.r,
                     geo=(Wo, Ho), out=T.view(lbn * Ho * Wo, self.r))
            prog = prog + [(len(srcs), 1, 0, 0, 1, 0, 0)]
            srcs = srcs + [ops.asrc_nhwc(T)]
            bs.append(ops.bsrc(L.lora.sb_fwd))
        out = self._new(B, Ho, Wo, N, dtype=torch.float32 if out_fp32 else BF16)
        ops.gemm(srcs, bs, prog, lin=False, M=M, N=N, geo=(Wo, Ho), out=out.view(M, N), bias=L.bias,
                 rowvec=rowvec, residual=None if residual is None else residual.reshape(M, N),
                 round_bf16=out_fp32, dep_a_src=None if T is None else len(srcs) - 1)
        if save is not None:
            save.append(("conv3", name, xs if lbn == B else [x[:lbn] for x in xs], T, stride))
        return out

    def linear(self, name, xs, lora, residual=None, act=0, save=None):
        """nn.Linear / 1x1 conv over [M, C] matrices xs (channel concat) (+LoRA), fused epilogue."""
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
        if lora and L.lora is not None:
            T = self._new(Ml, self.r)
            srcs_l = srcs if Ml == M else [ops.asrc_mat(x[:Ml]) for x in xs]
            ops.gemm(srcs_l, [ops.bsrc(L.lora.a_fwd)], prog, lin=True, M=Ml, N=self.r, out=T)
            prog = prog + [(len(srcs), 1, 0, 0, 1, 0, 0)]
            srcs = srcs + [ops.asrc_mat(T)]   # Ml rows: tiles past them read zeros (TMA bounds)
            bs.append(ops.bsrc(L.lora.sb_fwd))
        out = self._new(M, N)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=N, out=out, bias=L.bias, residual=residual, act=act,
                 dep_a_src=None if T is None else len(srcs) - 1)
        if save is not None:
            save.append(("linear", name, xs if Ml == M else [x[:Ml] for x in xs], T))
        return out

    def linear_group(self, lead, x, lora, save=None):
        """The g Linear layers of a shared-input group (attn1 q/k/v, attn2 k/v) as ONE GEMM:
        out[M, g*C] = x @ [W_0; ...; W_g-1]^T, layer i's LoRA up-projection entering as a K block that
        only feeds its own C output columns.  Returns the g column views of out."""
        G = self.groups[lead]
        g, Cc, r = G.g, G.cout, self.r
        M = x.shape[0]
        Ml = self._lrows(M)
        srcs, bs = [ops.asrc_mat(x)], [ops.bsrc(G.w_stack)]
        prog = [(0, 0, 0, 0, G.cin // 64, 0, 0)]
        T = None
        bn = 160 if Cc % 160 == 0 else 64
        if lora and G.lora:
            T = self._new(Ml, g * r)
            ops.gemm([ops.asrc_mat(x[:Ml])], [ops.bsrc(G.a_stack)], prog, lin=True, M=Ml, N=g * r, out=T)
            srcs.append(ops.asrc_mat(T))
            bs.append(ops.bsrc(G.sb_stack))
            prog = prog + [(1, 1, 0, 0, 1, i * r, 0, i * Cc, (i + 1) * Cc) for i in range(g)]
        out = self._new(M, g * Cc)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=g * Cc, out=out, block_n=bn,
                 dep_a_src=None if T is None else 1)
        if save is not None:
            save.append(("lgroup", lead, x[:Ml], T))
        return [out[:, i * Cc:(i + 1) * Cc] for i in range(g)]

    def gn(self, name, xs, B, HW, eps, silu, save=None):
        L = self.layers[name]
        C = sum(x.shape[-1] for x in xs)
        out = self._new(B * HW, C)
        stats = self._new(B, self.cfg.norm_num_groups, 2, dtype=torch.float32)
        ops.groupnorm_fwd(xs[0], xs[1] if len(xs) > 1 else None, L.gamma, L.beta, eps, silu, out, stats,
                          B, HW, self.cfg.norm_num_groups)
        if save is not None:
            lb = self._lrows(B)
            save.append(("gn", name, xs if lb == B else [x[:lb * HW] for x in xs], stats[:lb], eps, silu, lb, HW))
        return out

    def ln(self, name, x, save=None):
        L = self.layers[name]
        out = torch.empty_like(x)
        stats = self._new(x.shape[0], 2, dtype=torch.float32)
        ops.layernorm_fwd(x, L.gamma, L.beta, out, stats)
        if save is not None:
            Ml = self._lrows(x.shape[0])
            save.append(("ln", name, x[:Ml], stats[:Ml]))
        return out

    def attention(self, q, k, v, B, Sq, Skv, save=None, heads=None):
        Hh = heads or self.cfg.num_heads
        D = q.shape[1] // Hh
        out = self._new(q.shape[0], q.shape[1])
        lse = self._new(B, Hh, Sq, dtype=torch.float32)
        ops.attn_fwd(q, k, v, out, lse, B, Hh, Sq, Skv, D, D ** -0.5)
        if save is not None:
            lb = self._lrows(B)
            save.append(("attn", q[:lb * Sq], k[:lb * Skv], v[:lb * Skv], out[:lb * Sq], lse[:lb], lb, Sq, Skv, Hh))
        return out

    # ------------------------------------------------------------------------------------
    # blocks (forward)
    # ------------------------------------------------------------------------------------
    def resnet(self, p, xs, st, lora, save):
        """xs: list of NHWC sources (skip concat = 2 sources).  Returns [B,H,W,Cout]."""
        B, H, W, _ = xs[0].shape
        HW = H * W
        cin = sum(x.shape[-1] for x in xs)
        cout = self.layers[p + ".conv1"].cout
        flat = [x.view(B * HW, x.shape[-1]) for x in xs]
        h = self.gn(p + ".norm1", flat, B, HW, 1e-5, True, save)
        if self._temb is not None:
            G = self.temb_group
            i = G.index[p + ".time_emb_proj"]
            out_all, T_all = self._temb
            tproj = out_all[:, G.offs[i]:G.offs[i + 1]]
            if save is not None:
                save.append(("linear", p + ".time_emb_proj", [st[:self._lrows(st.shape[0])]], T_all, i * self.r))
        else:
            tproj = self.linear(p + ".time_emb_proj", [st], lora, save=save)
        h = self.conv3(p + ".conv1", [h.view(B, H, W, cin)], lora, rowvec=tproj, save=save)
        h = self.gn(p + ".norm2", [h.view(B * HW, cout)], B, HW, 1e-5, True, save)
        if cin != cout:
            sc = self.linear(p + ".conv_shortcut", flat, lora, save=save).view(B, H, W, cout)
        else:
            sc = xs[0]
        return self.conv3(p + ".conv2", [h.view(B, H, W, cout)], lora, residual=sc, save=save)

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
        g = self.gn(p + ".norm", [xf], B, S, 1e-6, False, save)
        h = self.linear(p + ".proj_in", [g], lora, save=save)
        for d in range(self.cfg.depth(level)):
            t = p + f".transformer_blocks.{d}"
            n = self.ln(t + ".norm1", h, save)
            q, k, v = self.linear_group(t + ".attn1.to_q", n, lora, save=save)
            a = self.attention(q, k, v, B, S, S, save, heads)
            h = self.linear(t + ".attn1.to_out.0", [a], lora, residual=h, save=save)
            n = self.ln(t + ".norm2", h, save)
            q = self.linear(t + ".attn2.to_q", [n], lora, save=save)
            if self._ctxkv is not None:
                k, v, Tkv = self._ctxkv[t]
                if save is not None:
                    save.append(("lgroup", t + ".attn2.to_k", ctx[:self._lrows(ctx.shape[0])], Tkv))
            else:
                k, v = self.linear_group(t + ".attn2.to_k", ctx, lora, save=save)
            a = self.attention(q, k, v, B, S, ctx.shape[0] // B, save, heads)
            h = self.linear(t + ".attn2.to_out.0", [a], lora, residual=h, save=save)
            n = self.ln(t + ".norm3", h, save)
            u = self.linear(t + ".ff.net.0.proj", [n], lora, save=save)
            gg = self._new(M, u.shape[1] // 2)
            ops.geglu_fwd(u, gg)
            if save is not None:
                save.append(("geglu", u[:self._lrows(M)]))
            h = self.linear(t + ".ff.net.2", [gg], lora, residual=h, save=save)
        return self.linear(p + ".proj_out", [h], lora, residual=xf, save=save).view(B, H, W, C)

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
        holds views of the first b samples, so backward() is the student's backward."""
        cfg = self.cfg
        lora = lora and self.has_lora
        tape = [] if save else None
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
        self._temb = self.temb_all(st, lora) if self.temb_group is not None else None
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
        skips = [x]
        nb = len(cfg.block_out_channels)
        marks = []  # tape segment boundaries for the backward walk
        for i in range(nb):
            for j in range(cfg.layers_per_block):
                x = self._block(tape, marks, "res", f"down_blocks.{i}.resnets.{j}", [x], st, lora)
                if cfg.down_attn[i]:
                    x = self._block(tape, marks, "attn", f"down_blocks.{i}.attentions.{j}", x, ctx, lora)
                skips.append(x)
            if i < nb - 1:
                x = self._block(tape, marks, "down", f"down_blocks.{i}.downsamplers.0.conv", x, None, lora)
                skips.append(x)
        x = self._block(tape, marks, "res", "mid_block.resnets.0", [x], st, lora)
        x = self._block(tape, marks, "attn", "mid_block.attentions.0", x, ctx, lora)
        x = self._block(tape, marks, "res", "mid_block.resnets.1", [x], st, lora)
        for i in range(nb):
            for j in range(cfg.layers_per_block + 1):
                x = self._block(tape, marks, "res", f"up_blocks.{i}.resnets.{j}", [x, skips.pop()], st, lora)
                if cfg.up_attn[i]:
                    x = self._block(tape, marks, "attn", f"up_blocks.{i}.attentions.{j}", x, ctx, lora)
            if i < nb - 1:
                x = self._block(tape, marks, "up", f"up_blocks.{i}.upsamplers.0.conv", x, None, lora)
        Bx, Hx, Wx, Cx = x.shape
        g = self.gn("conv_norm_out", [x.view(Bx * Hx * Wx, Cx)], Bx, Hx * Wx, 1e-5, True, tape)
        eps = self.conv3("conv_out", [g.view(Bx, Hx, Wx, Cx)], False, out_fp32=True)
        if save:
            self.saved = (tape, marks, (self._lb[0], H, W))
        return eps

    def _block(self, tape, marks, kind, name, x, aux, lora):
        start = len(tape) if tape is not None else 0
        if kind == "res":
            out = self.resnet(name, x, aux, lora, tape)
        elif kind == "attn":
            out = self.transformer(name, x, aux, lora, tape)
        elif kind == "down":
            out = self.conv3(name, [x], lora, stride=2, save=tape)
        else:  # up: nearest 2x then conv
            B, H, W, C = x.shape
            xu = self._new(B, 2 * H, 2 * W, C)
            ops.upsample2x_fwd(x, xu)
            out = self.conv3(name, [xu], lora, save=tape)
        if tape is not None:
            marks.append((kind, name, start, len(tape)))
        return out

    # ------------------------------------------------------------------------------------
    # backward primitives
    # ------------------------------------------------------------------------------------
    def _lora_wgrads(self, L, P_list, dy_mat, T_mat, dt_mat, taps_desc, lin, geo, M, q_c0=0):
        """dB += s * dy^T T[:, q_c0:q_c0+r] ;  dA += dt^T x  (per source / tap group)."""
        lo = L.lora
        with UNetB200._Side(self, (dy_mat, T_mat, dt_mat, P_list)):
            ops.wgrad(ops.asrc_mat(dy_mat), ops.asrc_mat(T_mat), lo.gB, lin=True, M=M, os_row=self.r, os_col=1,
                      alpha=self.scale, q_c0=q_c0)
            ktot = lo.gA.shape[1]
            for (psrc, taps, offs) in P_list:
                ops.wgrad(psrc, taps_desc(dt_mat), lo.gA, lin=lin, M=M, geo=geo, taps=taps, tap_off=offs,
                          os_row=1, os_col=ktot)

    def linear_bwd(self, rec, dy, need_dx=True, accumulate=None):
        """rec = ("linear", name, xs, T[, q_c0]).  Returns dx [M, cin_total] (or None)."""
        _, name, xs, T = rec[:4]
        q_c0 = rec[4] if len(rec) > 4 else 0
        L = self.layers[name]
        M = dy.shape[0]
        srcs, bs = [ops.asrc_mat(dy)], None
        dt = None
        if T is not None:
            dt = self._new(M, self.r)
            ops.gemm([ops.asrc_mat(dy)], [ops.bsrc(L.lora.sb_t)], [(0, 0, 0, 0, L.cout // 64, 0, 0)],
                     lin=True, M=M, N=self.r, out=dt)
            P_list, coff = [], 0
            for x in xs:
                P_list.append((ops.asrc_mat(x), ((0, 0),), (coff,)))
                coff += x.shape[1]
            self._keep.extend(xs)
            self._lora_wgrads(L, P_list, dy, T, dt, ops.asrc_mat, True, (1, 1), M, q_c0=q_c0)
        if not need_dx:
            return None
        prog = [(0, 0, 0, 0, L.cout // 64, 0, 0)]
        bs = [ops.bsrc(L.w_t)]
        if dt is not None:
            srcs.append(ops.asrc_mat(dt))
            bs.append(ops.bsrc(L.lora.a_t))
            prog.append((1, 1, 0, 0, 1, 0, 0))
        dx = self._new(M, L.cin)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=L.cin, out=dx, residual=accumulate,
                 dep_a_src=None if dt is None else 1)
        return dx

    def linear_group_bwd(self, rec, dpk, need_dx=True):
        """rec = ("lgroup", lead, x, T); dpk [M, g*C] = the g output gradients side by side.
        Returns dx [M, cin] (or None): ONE dgrad GEMM over K = g*C (+ the g LoRA blocks)."""
        _, lead, x, T = rec
        G = self.groups[lead]
        g, Cc, r = G.g, G.cout, self.r
        M = dpk.shape[0]
        dT = None
        if T is not None:
            dT = self._new(M, g * r)
            prog = [(0, 0, 0, 0, Cc // 64, i * Cc, 0, i * r, (i + 1) * r) for i in range(g)]
            ops.gemm([ops.asrc_mat(dpk)], [ops.bsrc(G.sbt_stack)], prog, lin=True, M=M, N=g * r, out=dT,
                     block_n=64)
            with UNetB200._Side(self, (dpk, T, dT, x)):
                for i, L in enumerate(G.layers):
                    ops.wgrad(ops.asrc_mat(dpk[:, i * Cc:(i + 1) * Cc]), ops.asrc_mat(T), L.lora.gB, lin=True,
                              M=M, os_row=r, os_col=1, alpha=self.scale, q_c0=i * r)
                    ops.wgrad(ops.asrc_mat(x), ops.asrc_mat(dT), L.lora.gA, lin=True, M=M, os_row=1,
                              os_col=G.cin, q_c0=i * r)
        if not need_dx:
            return None
        srcs, bs = [ops.asrc_mat(dpk)], [ops.bsrc(G.w_t_cat)]
        prog = [(0, 0, 0, 0, g * Cc // 64, 0, 0)]
        if dT is not None:
            srcs.append(ops.asrc_mat(dT))
            for i, L in enumerate(G.layers):
                bs.append(ops.bsrc(L.lora.a_t))
                prog.append((1, 1 + i, 0, 0, 1, i * r, 0))
        dx = self._new(M, G.cin)
        ops.gemm(srcs, bs, prog, lin=True, M=M, N=G.cin, out=dx, dep_a_src=None if dT is None else 1)
        return dx

    def conv3_bwd(self, rec, dy, need_dx=True, accumulate=None):
        """rec = ("conv3", name, xs, T, stride); dy [B,Ho,Wo,N].  Returns dx [B,H,W,cin_total]."""
        _, name, xs, T, stride = rec
        L = self.layers[name]
        B, Ho, Wo, N = dy.shape
        M = B * Ho * Wo
        geo = (Wo, Ho)
        dy_m = dy.view(M, N)
        dt = None
        if T is not None:
            dt = self._new(B, Ho, Wo, self.r)
            ops.gemm([ops.asrc_mat(dy_m)], [ops.bsrc(L.lora.sb_t)], [(0, 0, 0, 0, N // 64, 0, 0)],
                     lin=True, M=M, N=self.r, out=dt.view(M, self.r))
            P_list = []
            if stride == 1:
                coff = 0
                for x in xs:
                    P_list.append((ops.asrc_nhwc(x), TAPS3, [t * L.cin + coff for t in range(9)]))
                    coff += x.shape[-1]
            else:
                x = xs[0]
                for p in range(2):
                    for q in range(2):
                        taps, offs = [], []
                        for kh in range(3):
                            for kw in range(3):
                                if _S2[kh][0] == p and _S2[kw][0] == q:
                                    taps.append((_S2[kw][1], _S2[kh][1]))
                                    offs.append((kh * 3 + kw) * L.cin)
                        P_list.append((ops.asrc_nhwc(x[:, p::2, q::2, :]), taps, offs))
            lo = L.lora
            with UNetB200._Side(self, (dy, T, dt, xs)):
                ops.wgrad(ops.asrc_mat(dy_m), ops.asrc_mat(T.view(M, self.r)), lo.gB, lin=True, M=M,
                          os_row=self.r, os_col=1, alpha=self.scale)
                ktot = lo.gA.shape[1]
                for (psrc, taps, offs) in P_list:
                    ops.wgrad(psrc, ops.asrc_nhwc(dt), lo.gA, lin=False, M=M, geo=geo, taps=taps, tap_off=offs,
                              os_row=1, os_col=ktot)
        if not need_dx:
            return None
        cin = L.cin
        if stride == 1:
            srcs, bs = [ops.asrc_nhwc(dy)], [ops.bsrc(L.w_t)]
            prog = [(0, 0, -dw, -dh, N // 64, 0, t * N) for t, (dw, dh) in enumerate(TAPS3)]
            if dt is not None:
                srcs.append(ops.asrc_nhwc(dt))
                bs.append(ops.bsrc(L.lora.a_t))
                prog += [(1, 1, -dw, -dh, 1, 0, t * self.r) for t, (dw, dh) in enumerate(TAPS3)]
            dx = self._new(B, Ho, Wo, cin)
            ops.gemm(srcs, bs, prog, lin=False, M=M, N=cin, geo=geo, out=dx.view(M, cin),
                     residual=None if accumulate is None else accumulate.reshape(M, cin),
                     dep_a_src=None if dt is None else 1)
            return dx
        # stride 2: one launch per parity plane of dx
        H, W = 2 * Ho, 2 * Wo
        dx = self._new(B, H, W, cin)
        for p in range(2):
            for q in range(2):
                # x row 2i'+p receives dy row i'+s through kernel row kh: p=0 -> (kh=1, s=0);
                # p=1 -> (kh=0, s=+1), (kh=2, s=0)
                khs = [(1, 0)] if p == 0 else [(0, 1), (2, 0)]
                kws = [(1, 0)] if q == 0 else [(0, 1), (2, 0)]
                srcs, bs, prog, lprog = [ops.asrc_nhwc(dy)], [ops.bsrc(L.w_t)], [], []
                for kh, sh in khs:
                    for kw, sw in kws:
                        t = kh * 3 + kw
                        prog.append((0, 0, sw, sh, N // 64, 0, t * N))
                        lprog.append((1, 1, sw, sh, 1, 0, t * self.r))
                if dt is not None:
                    srcs.append(ops.asrc_nhwc(dt))
                    bs.append(ops.bsrc(L.lora.a_t))
                    prog += lprog
                plane = dx[:, p::2, q::2, :]
                acc = None if accumulate is None else accumulate[:, p::2, q::2, :]
                ops.gemm(srcs, bs, prog, lin=False, M=M, N=cin, geo=geo, out=plane, residual=acc,
                         out_strides=(plane.stride(2), plane.stride(1), plane.stride(0)), epi=(Wo, Wo * Ho),
                         dep_a_src=1 if (dt is not None and p == 0 and q == 0) else None)
        return dx

    def gn_bwd(self, rec, dy, add=None, colsum=None):
        _, name, xs, stats, eps, silu, B, HW = rec
        L = self.layers[name]
        dx1 = torch.empty_like(xs[0])
        dx2 = torch.empty_like(xs[1]) if len(xs) > 1 else None
        red = self._new(B, self.cfg.norm_num_groups, 2, dtype=torch.float32)
        ops.groupnorm_bwd(dy, xs[0], xs[1] if len(xs) > 1 else None, L.gamma, L.beta, eps, silu, stats, red,
                          add, dx1, dx2, B, HW, self.cfg.norm_num_groups, colsum=colsum)
        return dx1, dx2

    def ln_bwd(self, rec, dy, add=None):
        _, name, x, stats = rec
        dx = torch.empty_like(x)
        ops.layernorm_bwd(dy, x, self.layers[name].gamma, stats, add, dx)
        return dx

    def attn_bwd(self, rec, dout):
        _, q, k, v, out, lse, B, Sq, Skv, Hh = rec
        D = q.shape[1] // Hh
        Cc = q.shape[1]
        if q.stride(0) == 3 * Cc:     # self-attention: q/k/v are column views of one [M, 3C] matrix
            pk = self._new(q.shape[0], 3 * Cc)
            dq, dk, dv = pk[:, :Cc], pk[:, Cc:2 * Cc], pk[:, 2 * Cc:]
        elif k.stride(0) == 2 * Cc:   # cross-attention: k/v views of one [B*77, 2C] matrix
            dq = self._new(q.shape[0], Cc)
            pk = self._new(k.shape[0], 2 * Cc)
            dk, dv = pk[:, :Cc], pk[:, Cc:]
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
        delta = torch.empty_like(lse)
        ops.attn_bwd(q, k, v, out, dout, lse, delta, dq, dk, dv, B, Hh, Sq, Skv, D, D ** -0.5)
        return dq, pk

    # ------------------------------------------------------------------------------------
    # block backward (records were appended in forward order)
    # ------------------------------------------------------------------------------------
    def resnet_bwd(self, recs, dout, need_dx=True):
        """recs: [gn1, temb linear, conv1, gn2, (shortcut linear), conv2].  dout [B,H,W,Cout].
        Returns (dx1, dx2) for the (possibly concatenated) input sources."""
        has_sc = len(recs) == 6
        gn1, tlin, conv1, gn2 = recs[0], recs[1], recs[2], recs[3]
        conv2 = recs[-1]
        B, H, W, cout = dout.shape
        M = B * H * W
        dh2 = self.conv3_bwd(conv2, dout)                              # grad wrt silu(gn2(h1))
        # grad wrt h1 [M, cout]; its per-image column sums (= d tproj[b, n], the time-embedding
        # branch) are accumulated by the same kernel
        cs32 = self._new(B, cout, dtype=torch.float32)
        dh1, _ = self.gn_bwd(gn2, dh2.view(M, cout), colsum=cs32)
        # the time-embedding branch ends in LoRA weight gradients only: all of it on the side stream
        with UNetB200._Side(self, (cs32,)):
            drow = self._new(B, cout)
            ops.cast_f32_bf16(cs32, drow)
            self._keep.append(drow)
            self.linear_bwd(tlin, drow, need_dx=False)
        dh = self.conv3_bwd(conv1, dh1.view(B, H, W, cout), need_dx=need_dx)
        dsc = self.linear_bwd(recs[4], dout.view(M, cout), need_dx=need_dx) if has_sc else dout.view(M, cout)
        if not need_dx:
            return None, None
        return self.gn_bwd(gn1, dh.view(M, -1), add=dsc)

    def transformer_bwd(self, recs, dout):
        """recs order as appended by transformer(): gn, proj_in, depth x 13 block records, proj_out;
        dout [B,H,W,C]; returns dx [B,H,W,C]."""
        gn, pin, pout = recs[0], recs[1], recs[-1]
        blocks = recs[2:-1]
        assert len(blocks) % 13 == 0
        B, H, W, C = dout.shape
        M = B * H * W
        do = dout.view(M, C)
        dh = self.linear_bwd(pout, do)
        for bi in reversed(range(len(blocks) // 13)):
            (ln1, lqkv, at1, lo1, ln2, lq2, lkv2, at2, lo2, ln3, ff1, gegl, ff2) = blocks[13 * bi:13 * bi + 13]
            dh3 = dh
            dgg = self.linear_bwd(ff2, dh3)
            u = gegl[1]
            du = torch.empty_like(u)
            ops.geglu_bwd(dgg, u, du)
            dn3 = self.linear_bwd(ff1, du)
            dh2 = self.ln_bwd(ln3, dn3, add=dh3)
            da2 = self.linear_bwd(lo2, dh2)
            dq2, dkv2 = self.attn_bwd(at2, da2)
            with UNetB200._Side(self, (dkv2,)):     # feeds weight gradients only: off the dgrad chain
                self.linear_group_bwd(lkv2, dkv2, need_dx=False)
            dn2 = self.linear_bwd(lq2, dq2)
            dh1 = self.ln_bwd(ln2, dn2, add=dh2)
            da1 = self.linear_bwd(lo1, dh1)
            _, dqkv = self.attn_bwd(at1, da1)
            dn1 = self.linear_group_bwd(lqkv, dqkv)
            dh = self.ln_bwd(ln1, dn1, add=dh1)
        dg = self.linear_bwd(pin, dh)
        dx, _ = self.gn_bwd(gn, dg, add=do)
        return dx.view(B, H, W, C)

    def backward(self, d_eps, grad_ready=None):
        """d_eps: fp32 [B,H,W,4] gradient of the loss w.r.t. the student epsilon.
        Accumulates LoRA gradients into self.lora_grad (caller zeroes it between steps).
        grad_ready(offset): called (on the weight-gradient stream) after each block's backward with
        the flat-buffer offset from which every gradient element is final."""
        tape, marks, (B, H, W) = self.saved
        self._dkv_chunks = {}
        boffs = self.block_grad_offsets() if grad_ready is not None else None
        pending = []
        cfg = self.cfg
        c0 = cfg.block_out_channels[0]
        Lco = self.layers["conv_out"]
        dg = self._new(B, H, W, c0)
        ops.conv3x3_c4(d_eps, Lco.w_c4_t, None, dg, sgn=-1, round_in=False)
        d, _ = self.gn_bwd(tape[-1], dg.view(B * H * W, c0))
        d = d.view(B, H, W, c0)
        nb = len(cfg.block_out_channels)
        mi = len(marks) - 1
        dskips = []

        def pop():
            nonlocal mi
            # the block popped previously has been fully enqueued by now: its gradients are final once
            # the weight-gradient stream drains
            if grad_ready is not None and pending:
                off = boffs.get(pending.pop())
                if off is not None:
                    with UNetB200._Side(self, ()):
                        grad_ready(off)
            kind, name, s, e = marks[mi]
            mi -= 1
            pending.append(name)
            return kind, tape[s:e]

        # up path (reverse)
        for i in reversed(range(nb)):
            if i < nb - 1:
                _, recs = pop()
                dxu = self.conv3_bwd(recs[0], d)
                Bu, Hu, Wu, Cu = dxu.shape
                d = self._new(Bu, Hu // 2, Wu // 2, Cu)
                ops.upsample2x_bwd(dxu, d)
            for j in reversed(range(cfg.layers_per_block + 1)):
                if cfg.up_attn[i]:
                    _, recs = pop()
                    d = self.transformer_bwd(recs, d)
                _, recs = pop()
                d1, d2 = self.resnet_bwd(recs, d)
                Bc, Hc, Wc, _ = d.shape
                dskips.append(d2.view(Bc, Hc, Wc, -1))
                d = d1.view(Bc, Hc, Wc, -1)
        # mid
        for kind in ("res", "attn", "res"):
            k_, recs = pop()
            if k_ == "attn":
                d = self.transformer_bwd(recs, d)
            else:
                Bc, Hc, Wc, _ = d.shape
                d = self.resnet_bwd(recs, d)[0].view(Bc, Hc, Wc, -1)
        # down path (reverse); dskips is ordered s0..s11 reversed consumption -> s_last first
        def add_skip(dcur):
            ds = dskips_by_idx.pop()
            out = torch.empty_like(dcur)
            ops.add_bf16(dcur, ds, out)
            return out

        # up-path backward visited resnets in reverse, so dskips = [ds_0, ds_1, ..., ds_11]
        dskips_by_idx = dskips  # pop() from the end = highest skip index first
        for i in reversed(range(nb)):
            if i < nb - 1:
                d = add_skip(d)
                _, recs = pop()
                d = self.conv3_bwd(recs[0], d)
            for j in reversed(range(cfg.layers_per_block)):
                d = add_skip(d)
                if cfg.down_attn[i]:
                    _, recs = pop()
                    d = self.transformer_bwd(recs, d)
                _, recs = pop()
                first = (i == 0 and j == 0)
                Bc, Hc, Wc, _ = d.shape
                r = self.resnet_bwd(recs, d, need_dx=not first)
                if not first:
                    d = r[0].view(Bc, Hc, Wc, -1)
        if grad_ready is not None:
            with UNetB200._Side(self, ()):
                grad_ready(0)
        self._join_side()
        self.saved = None
