"""Attention layouts without a GPU.

Plan coverage: the SD1.5 and SDXL training steps are dry-run (ops record instead of launching) with
ops.attn_fwd / attn_bwd patched to record their tensor views.  Every launch is reduced to its layout
class, and the GPU case table of test_attn_gpu.py must cover each class, so a change to the UNet's
attention layouts fails here until a GPU case runs it.

Validation: pcm_attn_fwd / pcm_attn_bwd reject a layout no attention kernel can read (misaligned base
pointer, row stride not a multiple of 8 or shorter than H*D, empty dimension, a head size one direction
lacks) with an error naming the argument.  The fake pointers below are all rejected by that host-side
check, before any CUDA call, so nothing here can reach a launch."""
import pytest

import test_attn_gpu as attn_cases


def _dry_run_attention(cfg_name, batch, hw):
    """(kind, record) for every attention launch of one eager training step."""
    from pcm_b200 import config, ops, weights
    from pcm_b200.step import PCMTrainStep
    launches = []

    def fwd(q, k, v, out, lse, B, H, Sq, Skv, D, scale):
        launches.append(("fwd", dict(q=q, k=k, v=v, B=B, H=H, Sq=Sq, Skv=Skv, D=D)))

    def bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, B, H, Sq, Skv, D, scale):
        assert (dq.stride(0), dk.stride(0), dv.stride(0)) == (q.stride(0), k.stride(0), v.stride(0))
        launches.append(("bwd", dict(q=q, k=k, v=v, B=B, H=H, Sq=Sq, Skv=Skv, D=D)))

    old = (ops.DRY_RUN, ops.attn_fwd, ops.attn_bwd)
    ops.DRY_RUN, ops.attn_fwd, ops.attn_bwd = [], fwd, bwd
    try:
        cfg = getattr(config, cfg_name)
        st = PCMTrainStep(cfg, weights.synthetic_state_dict(cfg, 0), "cpu", batch=batch, height=hw,
                          width=hw, multiphase=4)
        launches.clear()
        st.run_eager()
    finally:
        ops.DRY_RUN, ops.attn_fwd, ops.attn_bwd = old
    return launches


def _layout(r):
    """(layout, chunk window position) of one launch's q / k / v views."""
    q, k, v, C = r["q"], r["k"], r["v"], r["H"] * r["D"]
    ldq, ldk, ldv = q.stride(0), k.stride(0), v.stride(0)
    if ldq == ldk == ldv == 3 * C and q.untyped_storage().data_ptr() == k.untyped_storage().data_ptr() \
            and k.storage_offset() == q.storage_offset() + C and v.storage_offset() == k.storage_offset() + C:
        return "fused", None
    if ldq == C and ldk == ldv > 2 * C and v.storage_offset() == k.storage_offset() + C:
        off = k.storage_offset() % ldk
        return "chunk", "first" if off == 0 else "last" if off + 2 * C == ldk else "interior"
    if ldq == ldk == ldv == C:
        return "dense", None
    raise AssertionError(f"unrecognised attention layout: ld {ldq}/{ldk}/{ldv}, C {C}")


def _plan_classes(launches):
    """Layout classes (d, Sq, Skv, layout, window position, merged) of a step's launches.  A backward
    is paired with the forward that made its q (the backward runs on a row slice of it); merged = the
    forward ran on more samples.  A forward without a backward covers both merged values."""
    fwds, last = [], {}     # [key, batch, has a backward]; q address -> latest forward from it
    classes = set()
    for kind, r in launches:
        key = (r["D"], r["Sq"], r["Skv"]) + _layout(r)
        if kind == "fwd":
            last[r["q"].data_ptr()] = len(fwds)
            fwds.append([key, r["B"], False])
        else:
            f = fwds[last[r["q"].data_ptr()]]
            assert f[0] == key and f[1] >= r["B"]
            f[2] = True
            classes.add(key + (f[1] > r["B"],))
    return classes, {f[0] for f in fwds if not f[2]}


@pytest.mark.parametrize("cfg_name,batch,hw", [("SD15", 8, 64), ("SDXL", 2, 128)])
def test_gpu_cases_cover_the_steps_attention_layouts(cfg_name, batch, hw):
    launches = _dry_run_attention(cfg_name, batch, hw)
    assert any(k == "bwd" for k, _ in launches)
    classes, fwd_only = _plan_classes(launches)
    covered = {attn_cases.layout_class(c) for c in attn_cases.CASES}
    missing = sorted(classes - covered, key=str)
    assert not missing, f"{cfg_name}: attention layouts no case of test_attn_gpu.py runs: {missing}"
    covered_fwd = {c[:-1] for c in covered}
    missing = sorted(fwd_only - covered_fwd, key=str)
    assert not missing, f"{cfg_name}: forward-only attention layouts no GPU case runs: {missing}"


# ---------------------------------------------------------------------------------------------
# host-side validation of pcm_attn_fwd / pcm_attn_bwd
# ---------------------------------------------------------------------------------------------
BASE = 1 << 40          # fake, 16-byte aligned device addresses: the check rejects before any use


def _fwd(lib, B=2, H=2, Sq=64, Skv=64, D=64, ld=(128, 128, 128, 128), q=BASE, k=BASE + 4096,
         v=BASE + 8192, out=BASE + 12288):
    return lib.pcm_attn_fwd(q, k, v, out, BASE + 16384, B, H, Sq, Skv, D, *ld, 0.125, None)


def _bwd(lib, B=2, H=2, Sq=64, Skv=64, D=64, ld=(128, 128, 128, 128), **ptrs):
    names = ["q", "k", "v", "o", "dout", "dq", "dk", "dv"]
    p = {n: BASE + 4096 * i for i, n in enumerate(names)}
    p.update(ptrs)
    return lib.pcm_attn_bwd(p["q"], p["k"], p["v"], p["o"], p["dout"], BASE + 65536, BASE + 69632,
                            p["dq"], p["dk"], p["dv"], B, H, Sq, Skv, D, *ld, 0.125, None)


@pytest.fixture(scope="module")
def lib():
    from pcm_b200 import _lib
    return _lib.lib()


def _rejects(lib, rc, msg):
    assert rc != 0
    assert lib.pcm_last_error().decode() == msg


@pytest.mark.parametrize("name", ["q", "k", "v", "out"])
def test_fwd_rejects_misaligned_pointer(lib, name):
    _rejects(lib, _fwd(lib, **{name: BASE + 8 * 4096 + 8}), f"attention: {name} is not 16-byte aligned")


@pytest.mark.parametrize("name", ["q", "k", "v", "o", "dout", "dq", "dk", "dv"])
def test_bwd_rejects_misaligned_pointer(lib, name):
    _rejects(lib, _bwd(lib, **{name: BASE + 16 * 4096 + 2}), f"attention: {name} is not 16-byte aligned")


@pytest.mark.parametrize("call", [_fwd, _bwd])
@pytest.mark.parametrize("i,name", list(enumerate(["ldq", "ldk", "ldv", "ldo"])))
def test_rejects_bad_row_stride(lib, call, i, name):
    ld = [128] * 4
    ld[i] = 132
    _rejects(lib, call(lib, ld=tuple(ld)), f"attention: {name} = 132 is not a multiple of 8")
    ld[i] = 120
    _rejects(lib, call(lib, ld=tuple(ld)), f"attention: {name} = 120 is less than H*D = 128")


@pytest.mark.parametrize("call", [_fwd, _bwd])
@pytest.mark.parametrize("name", ["B", "H", "Sq", "Skv"])
def test_rejects_empty_dimension(lib, call, name):
    _rejects(lib, call(lib, **{name: 0}), f"attention: {name} = 0 must be >= 1")


@pytest.mark.parametrize("call", [_fwd, _bwd])
@pytest.mark.parametrize("D", [0, 4, 12, 104, 112, 136, 144, 168, 256])
def test_rejects_unsupported_head_dim(lib, call, D):
    ld = (max(8, 2 * D),) * 4
    _rejects(lib, call(lib, D=D, ld=ld),
             f"attention: head dim {D} is not supported (multiples of 8 up to 96, and 120, 128, 152, 160)")


def test_head_dim_table_matches_gpu_test():
    assert attn_cases.SUPPORTED_HEAD_DIMS == tuple(list(range(8, 97, 8)) + [120, 128, 152, 160])
