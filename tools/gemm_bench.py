"""Micro-benchmark of pcm_gemm on representative step shapes (CUDA events, L2-cold between runs
by rotating buffers).  Usage: python tools/gemm_bench.py [shape_index]"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pcm_b200 import ops

dev = torch.device("cuda")
BF = torch.bfloat16
SHAPES = [  # (kind, M|(B,H,W), K|Cin, N, residual)
    ("lin", 32768, 384, 2560, False),
    ("lin", 32768, 384, 320, True),
    ("lin", 32768, 320, 64, False),
    ("lin", 8192, 704, 640, True),
    ("lin", 2048, 1344, 1280, True),
    ("conv", (8, 64, 64), 320, 320, True),
    ("conv", (8, 32, 32), 640, 640, True),
    ("conv", (8, 16, 16), 1280, 1280, True),
    ("conv", (8, 8, 8), 1280, 1280, True),
    ("lin", 8192, 640, 5120, False),
    ("lin", 32768, 1280, 320, True),
    ("lin", 98304, 384, 320, True),
    ("lin", 98304, 384, 2560, False),
    ("lin", 24576, 704, 640, True),
    ("conv", (24, 64, 64), 320, 320, True),
]
sel = [int(a) for a in sys.argv[1:]] or range(len(SHAPES))
iters = int(os.environ.get("ITERS", "20"))
for si in sel:
    kind, Mx, K, N, res = SHAPES[si]
    nbuf = 4
    if kind == "lin":
        M = Mx
        xs = [torch.randn(M, K, device=dev).to(BF) for _ in range(nbuf)]
        w = (torch.randn(N, K, device=dev) * K ** -0.5).to(BF)
        prog = [(0, 0, 0, 0, K // 64, 0, 0)]
        Ktot = K
    else:
        B, H, W = Mx
        M = B * H * W
        xs = [torch.randn(B, H, W, K, device=dev).to(BF) for _ in range(nbuf)]
        w = (torch.randn(N, 9 * K, device=dev) * (9 * K) ** -0.5).to(BF)
        prog = [(0, 0, dw, dh, K // 64, 0, t * K) for t, (dw, dh) in enumerate(ops.TAPS3)]
        Ktot = 9 * K
    outs = [torch.empty(M, N, device=dev, dtype=BF) for _ in range(nbuf)]
    rs = [torch.randn(M, N, device=dev).to(BF) for _ in range(nbuf)] if res else [None] * nbuf
    bias = torch.randn(N, device=dev)

    def run(i):
        x = xs[i % nbuf]
        a = [ops.asrc_mat(x)] if kind == "lin" else [ops.asrc_nhwc(x)]
        ops.gemm(a, [ops.bsrc(w)], prog, lin=(kind == "lin"), M=M, N=N, geo=(1, 1) if kind == "lin" else (W, H),
                 out=outs[i % nbuf], bias=bias, residual=rs[i % nbuf])
    for i in range(3):
        run(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        run(i)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    fl = 2.0 * M * N * Ktot
    print(f"[{si}] {kind} M={M} K={Ktot} N={N} res={res} bn={ops.pick_block_n(M, N)}: {us:8.1f} us  {fl / us / 1e6:7.1f} TFLOP/s", flush=True)
