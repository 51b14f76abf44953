"""Timing of the VAE decode and of its wide-head attention kernel on H100; one JSON line per measurement.

  python tools/bench_vae.py                       # one GPU: decode at 1024^2, 2048^2, 3840^2 (product vs the unsplit compat
                                                  # decoder in fp16 on torch's kernels) and df_attn_wide_fwd vs
                                                  # F.scaled_dot_product_attention at the mid-block shapes
  torchrun --nproc-per-node N tools/bench_vae.py --split   # the product decode split over N GPUs (rank 0 prints)
  python tools/bench_vae.py --upcast --no-kernel   # the stock SDXL VAE (force_upcast) decoded with upcast=True, against the
                                                  # compat decoder under diffusers' upcast split (fp16 to the mid block, fp32
                                                  # after) on torch's kernels; --split works with it too

Every line carries the card's name, power limit and SM clock, read with nvidia-smi in the same run.  Decode times are CUDA
events around whole decode calls after warm-up (median of --iters), with torch.cuda.max_memory_allocated of each decode
(peak_mib; reset before it, so it includes the model's weights); kernel times are CUDA graphs of --launches back-to-back
launches, TFLOP/s from the shape (4 L^2 d, d = 512)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.nn import functional as F  # noqa: E402

SIZES = (1024, 2048, 3840)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    idx = torch.cuda.current_device()
    return q[idx] if idx < len(q) else (q[0] if q else "unknown")


def _time(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def _vae(seed=11, upcast=False):
    from distrifuser_b200.compat.vae import SD15_VAE, SDXL_VAE, AutoencoderKL
    torch.manual_seed(seed)
    return AutoencoderKL(**(SDXL_VAE if upcast else SD15_VAE)).to("cuda", torch.float16).eval()


def _timed(row, key, fn, iters):
    """row[key + "_ms"] and row[key + "_peak_mib"] of fn, or "out of memory"."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    try:
        with torch.no_grad():
            row[key + "_ms"] = round(_time(fn, iters), 2)
        row[key + "_peak_mib"] = round(torch.cuda.max_memory_allocated() / 2 ** 20)
    except torch.cuda.OutOfMemoryError:
        row[key + "_ms"] = "out of memory"
    torch.cuda.empty_cache()


def bench_decode(px, iters, split, upcast):
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP, apply_upcast_split
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(height=px, width=px, split_batch=False)
    z = torch.randn(1, 4, px // 8, px // 8, generator=torch.Generator().manual_seed(5)).to("cuda", torch.float16)
    row = dict(what="decode_upcast" if upcast else "decode", px=px, world=cfg.world_size)
    pp = DistriAutoencoderKLPP(_vae(upcast=upcast), cfg, upcast=upcast)
    _timed(row, "product", lambda: pp.decode(z), iters)
    pp.close()
    del pp
    if not split:
        base = _vae(upcast=upcast)
        if upcast:
            apply_upcast_split(base)
        _timed(row, "torch_upcast_split" if upcast else "torch_fp16", lambda: base.decode(z), iters)
        del base
    torch.cuda.empty_cache()
    return row


def bench_kernel(L, launches):
    from distrifuser_b200 import _lib
    lib = _lib.lib()
    D = 512
    q = torch.randn(1, L, D, device="cuda", dtype=torch.float16)
    kv = torch.randn(1, L, 2 * D, device="cuda", dtype=torch.float16)
    out = torch.empty_like(q)
    lens, ranks = _lib.int32_array([L]), _lib.int32_array(range(8))

    def ours():
        _lib.check(lib.df_attn_wide_fwd(_lib.null_comm(), q.data_ptr(), kv.data_ptr(), out.data_ptr(), None, 1, L, lens, D,
                                        D, 2 * D, D, 1, 0, ranks, 0, 0, 0.0, torch.cuda.current_stream().cuda_stream),
                   "df_attn_wide_fwd")

    k, v = kv[..., :D].unsqueeze(1), kv[..., D:].unsqueeze(1)
    qh = q.unsqueeze(1)

    def sdpa():
        F.scaled_dot_product_attention(qh, k, v)

    flops = 4.0 * L * L * D
    row = dict(what="wide_attention", L=L)
    for name, fn in (("df_attn_wide_fwd", ours), ("sdpa", sdpa)):
        try:
            fn()
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(launches):
                    fn()
            ms = _time(g.replay, 3) / launches
            row[f"{name}_ms"] = round(ms, 3)
            row[f"{name}_tflops"] = round(flops / ms / 1e9, 1)
        except RuntimeError as e:                                    # e.g. no SDPA backend for this head width / length
            row[f"{name}_ms"] = f"failed: {str(e).splitlines()[0][:120]}"
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default=",".join(map(str, SIZES)))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--launches", type=int, default=4)
    ap.add_argument("--split", action="store_true", help="under torchrun: the product decode only, over every rank")
    ap.add_argument("--no-kernel", action="store_true")
    ap.add_argument("--upcast", action="store_true", help="the SDXL VAE with fp32 up blocks (DistriAutoencoderKLPP(upcast=True))")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vae measures on a GPU"
    sizes = [int(s) for s in a.sizes.split(",")]
    info = card()
    rank0 = int(os.environ.get("RANK", "0")) == 0
    for px in sizes:
        row = bench_decode(px, a.iters, a.split, a.upcast)
        if rank0:
            print(json.dumps(dict(row, card=info)), flush=True)
    if not a.split and not a.no_kernel:
        for px in sizes:
            print(json.dumps(dict(bench_kernel((px // 8) ** 2, a.launches), card=info)), flush=True)


if __name__ == "__main__":
    main()
