"""pcm_gemm / pcm_wgrad at the tile, ring and epilogue edges the production table cannot reach: synthetic
launches (tests/gemm_cases.py) through the same materialise / reference / check / guards as
test_gemm_prod_gpu.py."""
import itertools

import pytest

import gemm_cases
import gemm_spec as G
from gemm_cases import build, conv3x3_spec, dgrad2_spec, empty, linear_spec, restore, run, run_and_check, stride2_spec, wgrad_spec

pytestmark = pytest.mark.gpu
GEOMETRIES = [(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (128, 128), (8, 16), (16, 8), (4, 32)]


def linear(M, K, N, **kw):
    """linear_spec with a gutter after every output row, and no residual unless asked."""
    kw.setdefault("residual", False)
    return linear_spec(M, K, N, gutter=8, **kw)


def stages(block_n):
    """The ring depth launch_gemm derives for a tile width."""
    return min(8, (227 * 1024 - 512 - 1024 - 2 * 64 * 32 * 4) // (128 * 64 * 2 + block_n * 128))


@pytest.mark.parametrize("rank", [0, 24], ids=["plain", "narrow"])
@pytest.mark.parametrize("bn", range(32, 257, 32))
def test_every_block_n_at_its_n_edges(cuda, bn, rank):
    for N in (bn - 8, bn, bn + 8, bn + 13):
        run(linear(257, 128, N, block_n=bn, rank=rank, residual=True), cuda, N)


@pytest.mark.parametrize("M", [1, 127, 128, 129, 255, 257, "one tile more than the grid"])
def test_m_edges(cuda, M):
    M = 128 * G.num_sms() + 1 if isinstance(M, str) else M
    run(linear(M, 128, 64, block_n=64, residual=True), cuda, M)


@pytest.mark.parametrize("bn", range(32, 257, 32))
def test_ring_wrap(cuda, bn):
    S = stages(bn)
    for nkb in sorted({1, S - 1, S, S + 1, 2 * S + 1}):
        run(linear(300, 64 * nkb, bn + 8, block_n=bn), cuda, nkb)


@pytest.mark.parametrize("nkb,ks", [(10, 4), (5, 7), (9, 2), (16, 16)])
@pytest.mark.parametrize("N", [64, 100, 61])
def test_split_k(cuda, nkb, ks, N):
    for out, act in (("bf16", 0), ("fp32", 1), ("round", 0)):
        spec = linear(130, 64 * nkb, N, block_n=64, ksplit=ks, rowvec=True, residual=True, act=act, out=out, alpha=0.5)
        assert G.resolved_ksplit(spec["desc"]) > 1
        run(spec, cuda, nkb)


def test_a_split_too_short_to_run_is_an_ordinary_launch(cuda):
    spec = linear(200, 64, 64, ksplit=4, residual=True)
    assert G.resolved_ksplit(spec["desc"]) == 1
    run(spec, cuda)


@pytest.mark.parametrize("M,N", [(48, 24), (48, 40), (300, 168)])
@pytest.mark.parametrize("out", ["bf16", "fp32", "round"])
def test_every_epilogue_combination(cuda, M, N, out):
    for bias, rowvec, residual, act, alpha in itertools.product((0, 1), (0, 1), (0, 1, 2), (0, 1), (1.0, 0.25)):
        if residual == 2 and out != "bf16":
            continue                                       # in place needs a bf16 destination
        run(linear(M, 128, N, block_n=64, bias=bias, rowvec=rowvec, residual=residual == 1, inplace=residual == 2,
                   act=act, alpha=alpha, out=out), cuda, bias + 2 * rowvec)


@pytest.mark.parametrize("W,H", GEOMETRIES)
def test_conv_geometries(cuda, W, H):
    """3x3, stride 2 through parity planes, and its dgrad into one strided parity plane (the other three planes
    and the channel gutter are guarded).  B = 3 at the small images: the last 128-row tile leaves the batch."""
    B = 3 if W * H <= 1024 else 1
    run(conv3x3_spec(B, H, W, 64, 72, rowvec=True, residual=True), cuda, W)
    run(stride2_spec(B=B, H=H, W=W), cuda, H)
    for p, q in itertools.product(range(2), range(2)):
        run(dgrad2_spec(p, q, B=B, H=H, W=W, rank=24 * (p == q)), cuda, 2 * p + q)


@pytest.mark.parametrize("window", [(320, 0), (320, 128), (320, 192)], ids=["first", "interior", "last"])
def test_a_source_column_windows(cuda, window):
    run(linear(200, 128, 96, window=window), cuda)


@pytest.mark.parametrize("ranged", [None, (128, 256)], ids=["all columns", "middle N tile"])
@pytest.mark.parametrize("dep", [False, True])
@pytest.mark.parametrize("Ml", [256, 200])
def test_adapter_on_the_leading_rows(cuda, Ml, dep, ranged):
    """Ml a multiple of 128: the adapter K blocks of later M tiles are skipped (m_hi); otherwise TMA zero fill.
    Ranged: three N tiles, the adapter feeding only the middle one, so tiles fall outside the range on both
    sides and outside the rows.  dep: the down-projection runs immediately before, its output poisoned until then."""
    for rank in (8, 64, 152):
        run(linear(600, 192, 384, block_n=128, rank=rank, Ml=Ml, dep=dep, ranged=ranged), cuda, rank)


def test_max_sources_and_program_entries(cuda):
    from pcm_b200 import _lib

    def fn(ops):
        a = [ops.asrc_mat(empty((300, 64))) for _ in range(_lib.MAX_ASRC)]
        b = [ops.bsrc(empty((96, 64 * _lib.MAX_PROG))) for _ in range(_lib.MAX_BSRC)]
        prog = [(i % _lib.MAX_ASRC, i % _lib.MAX_BSRC, 0, 0, 1, 0, 64 * i) for i in range(_lib.MAX_PROG)]
        ops.gemm(a, b, prog, lin=True, M=300, N=96, out=empty((300, 96)), block_n=96)
    run(build(fn), cuda)


def _wgrad_both_ways(spec, cuda, seed):
    T = G.materialise(spec, cuda, seed)
    before = G.snapshot(T)
    run_and_check(spec, T, before)                       # unordered atomics
    restore(T, before)
    run_and_check(spec, T, before, sem=True)             # ordered by the semaphores
    assert not T.sem.any()


@pytest.mark.parametrize("M", [1, 127, 129, 1000])
@pytest.mark.parametrize("Cp", [64, 320, 1280])
def test_wgrad_linear_edges(cuda, M, Cp):
    slices = [(8, 0), (24, 0), (48, 0), (64, 0), (128, 64), (192, 128), (152, 128)]
    for (qC, q_c0), ks in zip(slices, itertools.cycle([0, 1, 100])):
        _wgrad_both_ways(wgrad_spec(True, M=M, Cp=Cp, qC=qC, q_c0=q_c0, ksplit=ks), cuda, qC)


@pytest.mark.parametrize("W,H", GEOMETRIES)
def test_wgrad_conv_taps(cuda, W, H):
    B = 3 if W * H <= 1024 else 1
    for (qC, q_c0), ks in zip(((64, 0), (88, 64)), (0, 100)):
        _wgrad_both_ways(wgrad_spec(False, B=B, H=H, W=W, Cp=320, qC=qC, q_c0=q_c0, ksplit=ks), cuda, W)


def test_report(cuda, capsys):
    with capsys.disabled():
        print("\n" + gemm_cases.report("GEMM edge cases (with the production classes when run in one session):"))
