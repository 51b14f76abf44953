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
    qh = q.float().view(b, lq, heads, d).transpose(1, 2)
    kh = k.float().view(b, -1, heads, d).transpose(1, 2)
    vh = v.float().view(b, -1, heads, d).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) / d ** 0.5
    o = torch.softmax(s, -1) @ vh
    return o.transpose(1, 2).reshape(b, lq, Cq)
