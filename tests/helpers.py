"""Shared helpers of the GPU parity tests (test infrastructure)."""
from __future__ import annotations

import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub")):
    if p not in sys.path:
        sys.path.insert(0, p)


def align(x, a):
    return (x + a - 1) // a * a


class LoopbackArena:
    """One process, one GPU: an arena whose `n` ranks all alias this rank's memory.  Lets a single GPU exercise the
    slot addressing, banks, flags and epoch clock of the multi-rank kernels; the test writes the "peers'" data and
    flags itself."""

    def __init__(self, n: int, slot_bytes: list[int], rank: int = 0, device="cuda"):
        from distrifuser_b200 import _lib
        self.lib = _lib.lib()
        self.n, self.rank = n, rank
        self.slot_bytes = [align(s, 256) for s in slot_bytes]
        nt = len(slot_bytes)
        header = align(4 * nt * n, 1024)
        self.tensor_off, off = [], header
        for sb in self.slot_bytes:
            self.tensor_off.append(off)
            off += n * sb
        self.bank_stride = align(off - header, 1024)
        total = header + _lib.NBANKS * self.bank_stride
        ptr = C.c_void_p()
        _lib.check(self.lib.df_symm_alloc(total, C.byref(ptr), None), "df_symm_alloc")
        self.ptr = ptr.value
        from distrifuser_b200.utils import _Holder
        self.arena = torch.as_tensor(_Holder(self.ptr, total), device=device)
        self.flags = self.arena[: 4 * nt * n].view(torch.int32).view(nt, n)
        self.clock = torch.zeros(4, dtype=torch.int32, device=device)
        self.tickets = torch.zeros(nt + 2, dtype=torch.int32, device=device)
        c = _lib.DfComm()
        for i in range(n):
            c.base[i] = self.ptr
            c.flags[i] = self.ptr
        c.clock, c.tickets = self.clock.data_ptr(), self.tickets.data_ptr()
        c.bank_stride, c.world, c.rank = self.bank_stride, n, rank
        self.comm = c

    def slot(self, epoch: int, idx: int, src: int, nbytes: int, dtype=torch.float16):
        o = (epoch % 3) * self.bank_stride + self.tensor_off[idx] + src * self.slot_bytes[idx]
        return self.arena[o:o + nbytes].view(dtype)

    def set_clock(self, pub: int, rd: int):
        self.clock[0], self.clock[1] = pub, rd

    def close(self):
        torch.cuda.synchronize()
        self.arena = None
        self.flags = None
        self.lib.df_symm_free(self.ptr)


def sdpa_ref(q, k, v, heads):
    """fp32 reference of softmax(q k^T / sqrt(d)) v; q:[b,lq,C] k,v:[b,lk,C]."""
    b, lq, Cq = q.shape
    d = Cq // heads
    qh = q.float().reshape(b, lq, heads, d).transpose(1, 2)
    kh = k.float().reshape(b, -1, heads, d).transpose(1, 2)
    vh = v.float().reshape(b, -1, heads, d).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) / d ** 0.5
    o = torch.softmax(s, -1) @ vh
    return o.transpose(1, 2).reshape(b, lq, Cq)


def _sdpa_ref_chunked(q, k, v, heads, chunk=1800):
    """fp32 reference for shapes whose [heads, lq, lk] score tensor does not fit: q rows in chunks."""
    out = torch.empty(q.shape, dtype=torch.float32, device=q.device)
    for r0 in range(0, q.shape[1], chunk):
        out[:, r0:r0 + chunk] = sdpa_ref(q[:, r0:r0 + chunk], k, v, heads)
    return out


def _attn(q, kv, heads, comm=None, maps=None, nseg=1, own=0, idx=0, lseg=None, wait=0, no_ws=False, out=None, scale=0.0,
          ws=None, d=None):
    """df_attn_fwd on q:[b,lq,heads*d] and this rank's K/V segment kv:[b,lseg,2*heads*d] (any row pitches).  `out`: written in
    place (default: a new contiguous tensor).  `ws`: a caller-owned zeroed workspace (default: a fresh one of
    df_attn_workspace_bytes; no_ws: none, i.e. the static whole-unit schedule).  `d`: stored head width (default C / heads)."""
    from distrifuser_b200 import _lib
    b, lq, Cq = q.shape
    d = d or Cq // heads
    if out is None:
        out = torch.empty(q.shape, dtype=q.dtype, device=q.device)
    seg_rank = (C.c_int32 * 8)(*range(8))
    L = _lib.lib()
    if ws is None:
        # zeroed scratch: ticket counter of the dynamic schedule, partials of split units (no_ws: static whole-unit lists instead)
        ws_bytes = 0 if no_ws else L.df_attn_workspace_bytes(b, lq, lseg or kv.shape[1], nseg, heads, d)
        ws = torch.zeros(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
    else:
        ws_bytes = ws.numel()
    _lib.check(L.df_attn_fwd(comm or _lib.null_comm(), q.data_ptr(), kv.data_ptr(), out.data_ptr(), maps, b, lq,
                             lseg or kv.shape[1], heads, d, q.stride(1), kv.stride(1), out.stride(1), nseg, own,
                             seg_rank, idx, wait, scale, ws.data_ptr() if ws_bytes else None, ws_bytes,
                             torch.cuda.current_stream().cuda_stream), "df_attn_fwd")
    torch.cuda.synchronize()
    return out


def _gn_ref(x, G, w, b_, eps, mean, meansq, bessel=True, silu=False):
    B, Cc, H, W = x.shape
    x5 = x.float().view(B, G, Cc // G, H, W)
    var = meansq - mean * mean
    ne = (Cc // G) * H * W
    if bessel:
        var = var * (ne / (ne - 1))
    y = ((x5 - mean) / (var + eps).sqrt()).view(B, Cc, H, W) * w.float().view(1, -1, 1, 1) + b_.float().view(1, -1, 1, 1)
    return torch.nn.functional.silu(y) if silu else y


def _moments(x, G):
    B, Cc, H, W = x.shape
    x5 = x.float().view(B, G, Cc // G, H, W)
    return x5.mean(dim=[2, 3, 4], keepdim=True), (x5 * x5).mean(dim=[2, 3, 4], keepdim=True)


def _gn_call(x, G, w, b_, eps, mode, bessel, negfb, silu, comm, idx, off, sb, mask, addend=None, apitch=0):
    from distrifuser_b200 import _lib
    L = _lib.lib()
    B, Cc, H, W = x.shape
    y = torch.empty_like(x, memory_format=torch.channels_last)
    scratch = torch.zeros(L.df_groupnorm_scratch_bytes(B, G, H, W, Cc), dtype=torch.uint8, device="cuda")
    _lib.check(L.df_groupnorm_fwd(comm, x.data_ptr(), addend.data_ptr() if addend is not None else None, apitch, y.data_ptr(), w.data_ptr(), b_.data_ptr(), B, H, W, Cc, G, eps, mode,
                                  bessel, negfb, silu, idx, off, sb, mask, scratch.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream), "df_groupnorm_fwd")
    torch.cuda.synchronize()
    return y


def _close(out, ref, rel=2e-3, abs_=4e-3):
    """GEMM tolerance: fp16 storage of an fp32-accumulated result, |err| <= abs_ + rel * |ref|."""
    err = (out.float() - ref).abs()
    bad = err > (abs_ + rel * ref.abs())
    assert not bad.any(), f"max err {err.max().item():.4e} at ref {ref.flatten()[err.flatten().argmax()].item():.3f}; {int(bad.sum())} bad"


def psnr(a, ref, floor=1e-20):
    """PSNR of `a` against `ref` in dB, peak = max |ref| (the reference's metric, scripts/compute_metrics.py:62-79)."""
    mse = ((a - ref) ** 2).mean().item()
    return 10 * torch.log10(ref.abs().max() ** 2 / max(mse, floor)).item()


def check_parity(name, outs, want, ranks_identical=False):
    """Product eps predictions (per rank, per step) against golden or oracle ones (per step): fp16 with fp32 accumulation
    against fp32, on outputs of std ~0.35: mean |err| < 4e-3, max |err| < 4e-2 and PSNR > 45 dB every step.
    `ranks_identical`: every rank also holds rank 0's output bit for bit."""
    for r, per_rank in enumerate(outs):
        assert len(per_rank) == len(want), f"{name} rank{r}: {len(per_rank)} steps, want {len(want)}"
        for t, (a, b) in enumerate(zip(per_rank, want)):
            assert a.shape == b.shape
            err = (a - b).abs()
            p = psnr(a, b)
            assert err.mean().item() < 4e-3 and err.max().item() < 4e-2 and p > 45, \
                f"{name} rank{r} step{t}: mean {err.mean():.2e} max {err.max():.2e} psnr {p:.1f} dB"
    if ranks_identical:
        for r, per_rank in enumerate(outs[1:], 1):
            for t, (a, b) in enumerate(zip(per_rank, outs[0])):
                assert torch.equal(a, b), f"{name}: rank {r} differs from rank 0 at step {t}"
