"""Host-side launch-plan checks that need no GPU: the step is sequenced in DRY_RUN mode (ops record
instead of launching) and the recorded K programs / operand layouts are validated against the rules
the CUDA side enforces (pcm_gemm: gemm_tc.cu launch_gemm) - so a plan bug fails here, on CPU."""
import collections

import pytest
import torch


@pytest.fixture(scope="module")
def dry_step():
    from pcm_b200 import config, ops, weights
    from pcm_b200.step import PCMTrainStep
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        cfg = config.TINY
        sd = weights.synthetic_state_dict(cfg, 0)
        st = PCMTrainStep(cfg, sd, "cpu", batch=2, height=16, width=16, multiphase=4)
        ops.DRY_RUN.clear()
        st.run_eager()
        rec = list(ops.DRY_RUN)
    finally:
        ops.DRY_RUN = old
    return st, rec


def test_k_programs_are_valid(dry_step):
    from pcm_b200 import _lib
    _, rec = dry_step
    gemms = [r[1] for r in rec if r[0] == "gemm"]
    assert gemms
    ranged = 0
    for g in gemms:
        assert 1 <= g["num_a"] <= _lib.MAX_ASRC and 1 <= g["num_b"] <= _lib.MAX_BSRC
        assert 1 <= len(g["prog"]) <= _lib.MAX_PROG
        bn = g["bn"]
        assert 32 <= bn <= 256 and bn % 32 == 0
        has_range = False
        for e in g["prog"]:
            a_src, b_src, dw, dh, nch, a_c0, b_k0 = e[:7]
            assert 0 <= a_src < g["num_a"] and 0 <= b_src < g["num_b"] and nch >= 1
            assert a_c0 % 64 == 0 and b_k0 % 64 == 0
            assert a_c0 + 64 * nch <= g["a_C"][a_src] + 63, (e, g["a_C"])      # within the A channels
            assert b_k0 + 64 * nch <= g["b_K"][b_src], (e, g["b_K"])            # within the B rows' K
            assert g["b_N"][b_src] >= min(g["N"], g["b_N"][b_src])
            if len(e) > 7 and e[8]:
                n_lo, n_hi = e[7], e[8]
                has_range = True
                assert n_lo % bn == 0 and n_lo < n_hi <= g["N"]
                assert n_hi % bn == 0 or n_hi == g["N"]
        if has_range:
            ranged += 1
            assert g["ksplit"] == 1      # N-ranged programs are not split over K
    assert ranged > 0                    # the q/k/v and cross-attention k/v groups use them


def test_grouped_layers_read_one_stacked_operand(dry_step):
    st, rec = dry_step
    net = st.unet
    assert net.groups
    # the one forward operand that holds each layer, and the layer's first row in it
    owner = {L.name: (key, op, n0) for key, op in net.operands.items() for L, n0 in op.members}
    for lead, G in net.groups.items():
        assert G.g in (2, 3)
        # stacked frozen weights, stored K-blocked [K/64][N][64] (pcm_bsrc.kblocked): q / k / v as their own
        # operand, cross-attention k / v as consecutive rows of a context chunk
        key, op, n0 = owner[lead]
        if lead.endswith(".attn1.to_q"):
            assert key == lead and op.w.shape == (G.cin // 64, G.g * G.cout, 64)
        else:
            c, j = net.ctx_group.where[lead[:-len(".attn2.to_k")]]
            ch = net.ctx_group.chunks[c]
            assert key == ch.key and op.w.shape == (G.cin // 64, ch.n_total, 64) and n0 == 2 * j * G.cout
        for i, L in enumerate(G.layers):
            assert owner[L.name][0] == key and owner[L.name][2] == n0 + i * G.cout
        if G.lora:
            r = net.r
            assert G.a_stack.shape == (G.g * r, G.cin)
            assert G.sb_stack.shape == (G.g * G.cout, r)
            assert G.sbt_stack.shape == (G.g * r, G.cout)


def test_lora_operand_layout_is_a_partition(dry_step):
    """Every (A, s*B, (s*B)^T, A^T) copy occupies its own slice of lora_opnd; together they tile it."""
    st, _ = dry_step
    net = st.unet
    spans = []
    for L in net.lora_layers:
        lo = L.lora
        taps = L.k * L.k if L.kind == "conv" else 1
        na, nb = net.r * taps * L.cin, L.cout * net.r
        spans += [(lo.o_a_fwd, na), (lo.o_sb_fwd, nb), (lo.o_sb_t, nb), (lo.o_a_t, na)]
    spans.sort()
    pos = 0
    for off, n in spans:
        assert off == pos, (off, pos)
        pos += n
    assert pos == net.lora_opnd.numel()
    # the refresh table addresses exactly these slices
    tab = net.refresh_table.cpu()
    assert tab.shape[0] == len(net.lora_layers)
    for row, L in zip(tab.tolist(), net.lora_layers):
        lo = L.lora
        assert row[2:6] == [lo.o_a_fwd, lo.o_sb_fwd, lo.o_sb_t, lo.o_a_t]


def test_launch_census(dry_step):
    _, rec = dry_step
    c = collections.Counter(r[0] for r in rec)
    # one pass each of the PCM math kernels, one optimiser, one LoRA refresh
    for k in ("pcm_prepare", "pcm_teacher_step", "pcm_loss", "pcm_grad_sumsq", "pcm_adamw_clip", "pcm_lora_refresh"):
        assert c[k] == 1, (k, c[k])
    assert c["pcm_add_noise"] == 3
    assert c["gemm"] > c["wgrad"] > 0
    assert c["pcm_attn_bwd"] * 2 == c["pcm_attn_fwd"]      # merged student+teacher pass + target pass


def test_late_wait_launches_follow_their_producer(dry_step):
    """A GEMM launched with dep_a_src (late PDL wait) must come IMMEDIATELY after the launch that
    produced that source on the main stream (side-stream wgrads aside), and never after another
    late-wait GEMM - otherwise its early part could run before older inputs are complete."""
    _, rec = dry_step
    main = [r for r in rec if r[0] != "wgrad"]
    n_dep = 0
    for prev, cur in zip(main, main[1:]):
        if cur[0] != "gemm" or cur[1].get("dep") is None:
            continue
        n_dep += 1
        g = cur[1]
        assert prev[0] == "gemm", prev[0]
        assert prev[1].get("dep") is None, "two consecutive late-wait GEMMs"
        assert prev[1]["N"] == g["a_C"][g["dep"]], (prev[1]["N"], g["a_C"], g["dep"])
    assert n_dep > 100


def _dry(cfg_name, **kw):
    from pcm_b200 import config, ops, weights
    from pcm_b200.step import PCMTrainStep
    old = ops.DRY_RUN
    ops.DRY_RUN = []
    try:
        cfg = getattr(config, cfg_name)
        st = PCMTrainStep(cfg, weights.synthetic_state_dict(cfg, 0), "cpu", batch=2, height=16, width=16,
                          multiphase=4, **kw)
        ops.DRY_RUN.clear()
        st.run_eager()
        return st, collections.Counter(r[0] for r in ops.DRY_RUN), list(ops.DRY_RUN)
    finally:
        ops.DRY_RUN = old


def test_sdxl_shaped_plan():
    """SDXL-shaped network: transformer depth (1, 2, 3) -> 2*2 + 3*(2+1+... ) stacks; every K program valid;
    the text_time embedding adds its two Linear layers and one more sinusoid launch per pass."""
    from pcm_b200 import _lib, config
    st, c, rec = _dry("TINY_XL", num_ddim_timesteps=40)
    base, _, _ = _dry("TINY")
    cfg = config.TINY_XL
    # transformer blocks per pass: down (2 attn x depth) + mid + up (3 attn x depth), levels with attention only
    blocks = sum(2 * cfg.depth(i) for i in range(3) if cfg.down_attn[i]) + cfg.depth(2) + \
        sum(3 * cfg.depth(2 - i) for i in range(3) if cfg.up_attn[i])
    assert c["pcm_geglu_fwd"] == 2 * blocks               # merged student + teacher pass, target pass
    assert c["pcm_geglu_bwd"] == blocks
    assert c["pcm_timestep_embed"] == 4                   # (t, time_ids) x 2 passes
    for g in (r[1] for r in rec if r[0] == "gemm"):
        assert len(g["prog"]) <= _lib.MAX_PROG and g["num_b"] <= _lib.MAX_BSRC
        for e in g["prog"]:
            assert e[6] % 64 == 0                          # b_k0 on a K-block boundary (K-blocked weights)


def test_teacher_substeps_plan():
    """k teacher sub-steps: k - 1 extra frozen-teacher passes (batch 2B, no tape) and k substep launches."""
    _, c1, _ = _dry("TINY")
    _, c2, rec2 = _dry("TINY", teacher_substeps=2)
    assert c1["pcm_teacher_step"] == 1 and "pcm_teacher_substep" not in c1
    assert c2["pcm_teacher_substep"] == 2 and "pcm_teacher_step" not in c2
    assert c2["pcm_attn_fwd"] == c1["pcm_attn_fwd"] * 3 // 2      # 2 passes -> 3 passes
    assert c2["pcm_attn_bwd"] == c1["pcm_attn_bwd"]               # the backward is the student's only
    assert c2["wgrad"] == c1["wgrad"]
