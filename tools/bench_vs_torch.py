"""Library / eager-PyTorch context for the two hand-written kernels, at the SDXL shapes (same box, CUDA events, L2 flushed):
  * attention: df_attn_fwd vs torch F.scaled_dot_product_attention (what the reference calls, attn.py:153) on the same tensors;
  * GroupNorm: df_groupnorm_fwd vs the reference module's eager op sequence (groupnorm.py:38-41,58-72: two means, stack, var,
    normalise, affine) and vs torch.nn.functional.group_norm.
Informational; never a bench value."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from distrifuser_b200 import _lib  # noqa: E402

L = _lib.lib()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


print("== attention (fp16, non-causal)")
for name, (b, lq, lk, h, d) in {"1024^2 level1": (2, 4096, 4096, 10, 64), "1024^2 level2": (2, 1024, 1024, 20, 64),
                                "3840^2 n=4 level2": (1, 3600, 14400, 20, 64), "SD1.x level0 d=40": (2, 4096, 16384, 8, 40)}.items():
    Cq = h * d
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16)
    out = torch.empty_like(q)
    seg = (C.c_int32 * 8)(*range(8))
    st = torch.cuda.current_stream().cuda_stream

    ws_bytes = L.df_attn_workspace_bytes(b, lq, lk, 1, h, d)
    ws = torch.zeros(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")

    def ours():
        _lib.check(L.df_attn_fwd(_lib.null_comm(), q.data_ptr(), kv.data_ptr(), out.data_ptr(), None, b, lq, lk, h, d, q.stride(1),
                                 kv.stride(1), out.stride(1), 1, 0, seg, 0, 0, 0.0, ws.data_ptr() if ws_bytes else None, ws_bytes, st), "attn")
    qh = q.view(b, lq, h, d).transpose(1, 2)
    kh = kv[..., :Cq].reshape(b, lk, h, d).transpose(1, 2)
    vh = kv[..., Cq:].reshape(b, lk, h, d).transpose(1, 2)

    def sdpa():
        return F.scaled_dot_product_attention(qh, kh, vh)
    fl = 4.0 * b * lq * lk * Cq
    t1, t2 = timeit(ours), timeit(sdpa)
    print(f"{name:20s} ours {t1 * 1e3:8.1f} us {fl / t1 / 1e9:7.1f} TFLOP/s | torch SDPA {t2 * 1e3:8.1f} us {fl / t2 / 1e9:7.1f} TFLOP/s | x{t2 / t1:.2f}")

print("== GroupNorm (+SiLU), b=2")
for name, (Cc, hh, ww) in {"C=320 128x128": (320, 128, 128), "C=640 64x64": (640, 64, 64), "C=1280 32x32": (1280, 32, 32)}.items():
    b, G = 2, 32
    x = torch.randn(b, Cc, hh, ww, device="cuda", dtype=torch.float16)
    xcl = x.contiguous(memory_format=torch.channels_last)
    w = torch.randn(Cc, device="cuda", dtype=torch.float16)
    bb = torch.randn(Cc, device="cuda", dtype=torch.float16)
    y = torch.empty_like(xcl)
    scratch = torch.zeros(L.df_groupnorm_scratch_bytes(b, G, hh, ww, Cc), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def ours():
        _lib.check(L.df_groupnorm_fwd(_lib.null_comm(), xcl.data_ptr(), None, 0, y.data_ptr(), w.data_ptr(), bb.data_ptr(), b, hh, ww, Cc,
                                      G, 1e-5, 0, 1, 0, 1, 0, 0, 0, 1, scratch.data_ptr(), st), "gn")

    def reference_eager():        # groupnorm.py:37-41,58-72 (local statistics) followed by the block's SiLU
        x5 = x.view(b, G, Cc // G, hh, ww)
        m = x5.mean(dim=[2, 3, 4], keepdim=True)
        m2 = (x5 ** 2).mean(dim=[2, 3, 4], keepdim=True)
        sm = torch.stack([m, m2], 0)
        var = sm[1] - sm[0] ** 2
        ne = Cc // G * hh * ww
        var = var * (ne / (ne - 1))
        o = ((x5 - sm[0]) / (var + 1e-5).sqrt()).view(b, Cc, hh, ww)
        o = o * w.view(1, -1, 1, 1) + bb.view(1, -1, 1, 1)
        return F.silu(o)

    def torch_gn():
        return F.silu(F.group_norm(x, G, w, bb, 1e-5))
    nbytes = 4.0 * x.numel()
    t1, t2, t3 = timeit(ours), timeit(reference_eager), timeit(torch_gn)
    print(f"{name:16s} ours {t1 * 1e3:7.1f} us {nbytes / t1 / 1e6:7.0f} GB/s | reference eager ops {t2 * 1e3:7.1f} us | F.group_norm+silu {t3 * 1e3:7.1f} us | x{t2 / t1:.1f} / x{t3 / t1:.1f}")
