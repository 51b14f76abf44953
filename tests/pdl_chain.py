"""A fixed, seeded chain of the library's kernels, enqueued back to back on one stream without host synchronisation, each
reading what the previous one wrote: GEMM with the GEGLU epilogue -> add + LayerNorm -> GroupNorm (local statistics) ->
GroupNorm (synchronous exchange with a loopback peer) -> attention (split K/V plan) -> attention (dynamic plan) -> GEMM.
Saves every output to argv[1].  Run with DF_PDL=15 (programmatic dependent launch for every kernel family) and without:
the outputs must be bit-identical (test_kernel_configs_gpu.py)."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import LoopbackArena  # noqa: E402  (helpers also puts the repository root on sys.path)


def main(path):
    from distrifuser_b200 import _lib, ops
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    dev = "cuda"
    torch.manual_seed(50)
    # ---- every input, weight and scratch buffer first: the chain below launches nothing but the library's kernels
    M, K, D = 2048, 640, 1280
    x = torch.randn(M, K, device=dev).half()
    w1 = (torch.randn(2 * D, K, device=dev) / K ** 0.5).half()
    b1 = (0.5 * torch.randn(2 * D, device=dev)).half()
    block = ops.geglu_block(M, 2 * D, K)
    w1i, b1i = ops.geglu_interleave(w1, b1, block)
    res = torch.randn(M, D, device=dev).half()
    ln = torch.nn.LayerNorm(D).to(dev).half()
    with torch.no_grad():
        ln.weight.copy_(1 + 0.1 * torch.randn(D)); ln.bias.copy_(0.1 * torch.randn(D))
    B, H, W, G = 2, 32, 32, 32                                   # the [2048, 1280] rows as two 32 x 32 NHWC images
    gw = (1 + 0.1 * torch.randn(D, device=dev)).half()
    gb = (0.1 * torch.randn(D, device=dev)).half()
    gn_scratch = [torch.zeros(L.df_groupnorm_scratch_bytes(B, G, H, W, D), dtype=torch.uint8, device=dev) for _ in range(2)]
    nb, e = B * G * 8, 3
    arena = LoopbackArena(2, [nb], rank=0)
    peer = torch.stack([0.3 * torch.randn(B * G, device=dev), 1.0 + torch.rand(B * G, device=dev)], -1)
    arena.slot(e, 0, 1, nb, torch.float32).copy_(peer.flatten())
    arena.flags[0, 1] = e
    arena.set_clock(pub=e, rd=e)
    heads, d = 10, 64                                            # attention on the first 640 columns (row pitch 1280)
    Ca = heads * d
    plans = {"attn_split": (1, 256, 2048), "attn_dynamic": (2, 1024, 1024)}     # (b, lq, lk): 20 units in 2 parts / 160 units
    ws = {k: torch.zeros(L.df_attn_workspace_bytes(b, lq, lk, 1, heads, d), dtype=torch.uint8, device=dev) for k, (b, lq, lk) in plans.items()}
    assert ws["attn_split"].numel() > 1024 and ws["attn_dynamic"].numel() == 1024
    w2 = (torch.randn(640, Ca, device=dev) / Ca ** 0.5).half()
    b2 = torch.randn(640, device=dev).half()
    seg_rank = (C.c_int32 * 8)(*range(8))
    torch.cuda.synchronize()

    # ---- the chain
    out = {}
    out["geglu"] = ops.linear_geglu(x, w1i, b1i, block)
    out["sum"], out["ln"] = ops.add_layernorm(out["geglu"], res, ln)
    src = out["ln"]
    for name, mode in (("gn_local", 0), ("gn_exchange", 1)):
        y = torch.empty(M, D, device=dev, dtype=torch.float16)
        comm = arena.comm if mode else _lib.null_comm()
        _lib.check(L.df_groupnorm_fwd(comm, src.data_ptr(), None, 0, y.data_ptr(), gw.data_ptr(), gb.data_ptr(), B, H, W, D, G, 1e-5,
                                      mode, 0, 0, 1, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b11, gn_scratch[mode].data_ptr(), st),
                   "df_groupnorm_fwd")
        out[name] = src = y
    kv_all = out["ln"]                                           # K | V rows: [b, lk, 2 * 640] views of the LayerNorm output
    for name, (b, lq, lk) in plans.items():
        q = src.view(b, lq * M // (b * lq), D)[:, :lq, :Ca]
        kv = kv_all.view(b, -1, 2 * Ca)[:, :lk]
        o = torch.empty(b, lq, Ca, device=dev, dtype=torch.float16)
        _lib.check(L.df_attn_fwd(_lib.null_comm(), q.data_ptr(), kv.data_ptr(), o.data_ptr(), None, b, lq, lk, heads, d, q.stride(1),
                                 kv.stride(1), o.stride(1), 1, 0, seg_rank, 0, 0, 0.0, ws[name].data_ptr(), ws[name].numel(), st),
                   "df_attn_fwd")
        out[name] = o
    out["proj"] = ops.linear(out["attn_dynamic"], w2, b2)
    torch.cuda.synchronize()
    torch.save({"pdl": int(os.environ.get("DF_PDL", "0")), "out": {k: v.cpu() for k, v in out.items()}}, path)
    arena.close()


if __name__ == "__main__":
    main(sys.argv[1])
