"""Micro-benchmark of df_attn_fwd (fmha_fwd_kernel) at the SDXL self-attention shapes.  Default: a CUDA graph of `--launches`
back-to-back launches on ROTATING q / kv / out buffers (total footprint > L2), timed with CUDA events over 5 replays -- the
kernel's average duration as it runs inside the captured UNet step, without the host launch gaps that an eager
event-bracketed launch picks up for 20-us kernels.  `--eager` times single launches (L2 flushed);
`--profile` brackets a single launch with cudaProfilerStart/Stop for ncu."""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

SHAPES = {  # name: (b, lq, lkv, heads, d)
    "1024_l1": (2, 4096, 4096, 10, 64), "1024_l2": (2, 1024, 1024, 20, 64),
    "3840n4_l2": (1, 3600, 14400, 20, 64), "3840n4_l1": (1, 14400, 57600, 10, 64),
    "2048n2_l1": (1, 8192, 16384, 10, 64), "cross_l2": (2, 1024, 77, 20, 64), "cross_l1": (2, 4096, 77, 10, 64),
    "1024n4_l2": (1, 256, 1024, 20, 64), "1024n4_l1": (1, 1024, 4096, 10, 64), "1024n2_l2": (1, 512, 1024, 20, 64),
    "1024n2_l1": (1, 2048, 4096, 10, 64), "sd15_l0": (2, 4096, 16384, 8, 40), "sd15_l1": (2, 1024, 4096, 8, 80),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1024_l1,1024_l2,3840n4_l2,2048n2_l1")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--launches", type=int, default=0, help="launches per graph (0 = enough for a > 300 MB footprint, 8..64)")
    ap.add_argument("--eager", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--no-split", action="store_true", help="disable split-KV (A/B)")
    a = ap.parse_args()
    from distrifuser_b200 import _lib
    L = _lib.lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    seg = (C.c_int32 * 8)(*range(8))
    for name in a.shapes.split(","):
        b, lq, lk, h, d = SHAPES[name]
        Cq = h * d
        per_launch = (2 * b * lq * Cq + b * lk * 2 * Cq) * 2
        n = a.launches or max(8, min(64, int(3e8 // per_launch) + 1))
        if a.eager or a.profile:
            n = 1
        qs = [torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16) for _ in range(n)]
        kvs = [torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(n)]
        outs = [torch.empty_like(q) for q in qs]
        ws_bytes = 0 if a.no_split else L.df_attn_workspace_bytes(b, lq, lk, 1, h, d)
        ws = torch.zeros(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")

        def run(i=0):
            st = torch.cuda.current_stream().cuda_stream
            q, kv, out = qs[i], kvs[i], outs[i]
            _lib.check(L.df_attn_fwd(_lib.null_comm(), q.data_ptr(), kv.data_ptr(), out.data_ptr(), None, b, lq, lk, h, d,
                                     q.stride(1), kv.stride(1), out.stride(1), 1, 0, seg, 0, 0, 0.0,
                                     ws.data_ptr() if ws_bytes else None, ws_bytes, st), "df_attn_fwd")
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        fl = 4.0 * b * lq * lk * Cq
        if a.profile:
            flush.zero_()
            torch.cuda.synchronize()
            torch.cuda.profiler.start()
            run()
            torch.cuda.synchronize()
            torch.cuda.profiler.stop()
            continue
        if a.eager:
            ts = []
            for _ in range(a.iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); run(); e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ts.sort()
            ms = ts[len(ts) // 2]
            how = "eager, L2 flushed"
        else:
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                for i in range(n):
                    run(i)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for i in range(n):
                    run(i)
            for _ in range(2):
                g.replay()
            reps = 5
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps / n
            how = f"graph of {n} launches, rotating buffers"
        print(f"{name:10s} b={b} lq={lq} lkv={lk} h={h} d={d}: {ms * 1e3:9.1f} us  {fl / ms / 1e9:8.1f} TFLOP/s   ({how})", flush=True)
        del qs, kvs, outs


if __name__ == "__main__":
    main()
