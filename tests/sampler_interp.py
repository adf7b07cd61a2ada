"""Test-side torch semantics of the two sampler kernels behind ops._call (include/pcm_b200.h:
pcm_lora_fuse, pcm_sample_step), on top of tests/ops_interp.py, so that the HOST sequencing of
pcm_b200/sampling.py (fused inference net, fuse table, CFG batch layout, step coefficients) runs on CPU.
Test infrastructure only: nothing under pcm_b200/ imports this file."""
import ctypes

import torch

import ops_interp
from gemm_interp import BF16
from ops_interp import PcmCalls, _raw


def _bf16(ptr, n):
    return _raw(ptr, n, ctypes.c_uint16, torch.int16).view(BF16)


def fuse_rows(table_ptr, num_entries):
    """The pcm_lora_fuse table as dicts (field meanings: include/pcm_b200.h)."""
    tab = _raw(table_ptr, num_entries * 8, ctypes.c_int64, torch.int64).view(num_entries, 8).tolist()
    out = []
    for a_off, b_off, src, dst, n0n, kr, n, w0 in tab:
        out.append(dict(a_off=a_off, b_off=b_off, src=src, dst=dst, n0=n0n & 0xffffffff, ntot=n0n >> 32,
                        K=kr & 0xffffffff, r=kr >> 32, n=n, work_begin=w0))
    return out


class SamplerCalls(PcmCalls):
    def pcm_lora_fuse(self, master, table, num_entries, total_work, scale):
        """dst[n0+n, k] = bf16(src[n0+n, k] + scale * (B A)[n, k]) on K-blocked [K/64][N_total][64] operands."""
        work = 0
        for e in fuse_rows(table, num_entries):
            K, r, n, ntot, n0 = e["K"], e["r"], e["n"], e["ntot"], e["n0"]
            assert e["work_begin"] == work
            A = _raw(master + 4 * e["a_off"], r * K, ctypes.c_float, torch.float32).view(r, K)
            Bm = _raw(master + 4 * e["b_off"], n * r, ctypes.c_float, torch.float32).view(n, r)
            src = _bf16(e["src"], K * ntot).view(K // 64, ntot, 64)[:, n0:n0 + n]
            dst = _bf16(e["dst"], K * ntot).view(K // 64, ntot, 64)[:, n0:n0 + n]
            ba = (Bm.double() @ A.double()).float().view(n, K // 64, 64).permute(1, 0, 2)
            dst.copy_((src.float() + scale * ba).to(BF16))
            work += (n // 64) * (K // 64)
        assert work == total_work

    def pcm_sample_step(self, eps, x, out, out2, per, B, cfg, guidance, sa, ss, sap, ssp, pred_type):
        f = lambda p, rows: _raw(p, rows * per, ctypes.c_float, torch.float32).view(rows, per)  # noqa: E731
        if cfg:
            g = float(_raw(guidance, 1, ctypes.c_double, torch.float64)[0])
            e2 = f(eps, 2 * B).double()
            e = e2[:B] + g * (e2[B:] - e2[:B])
        else:
            e = f(eps, B).double()
        xv = f(x, B).double()
        if pred_type == 0:
            x0, pe = (xv - ss * e) / sa, e
        else:
            x0, pe = sa * xv - ss * e, sa * e + ss * xv
        y = (sap * x0 + ssp * pe).float()
        f(out, B).copy_(y)
        if out2:
            f(out2, B).copy_(y)


def install(monkeypatch):
    from pcm_b200 import ops
    ops_interp.install(monkeypatch)
    monkeypatch.setattr(ops, "_call", SamplerCalls())
