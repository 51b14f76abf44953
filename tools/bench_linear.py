"""df_linear_fwd (hand-written wgmma GEMM, csrc/linear.cu) vs torch F.linear (cuBLAS nvjet) at the Linear shapes of one SDXL
denoise step, and the fused GEGLU projection vs F.linear + df_geglu.  Timing: CUDA events around replays of a CUDA graph that cycles 6 distinct (input, weight) sets (weights stream from HBM as in the model, no host launch gaps).  Informational: it tells which
Linear kinds are worth enabling through DF_LINEAR (ops.py): its default, `geglu`, holds the kinds that beat cuBLAS here."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from distrifuser_b200 import ops  # noqa: E402

flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


NSETS = 6      # distinct (input, weight, bias) sets cycled inside one CUDA graph: every launch streams its weights from HBM,
               # as in the model (5 GB of weights per denoise step), and no host launch gap is timed


def timeit(make_fn, sets, reps=5):
    """make_fn(set) -> callable.  Average device time of one call inside a CUDA graph of len(sets) x 2 calls."""
    fns = [make_fn(s_) for s_ in sets]
    for f in fns:
        f()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for f in fns:
            f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(2):
            for f in fns:
                f()
    for _ in range(2):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps / (2 * len(fns))


res = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
T2, T1 = 2 * (res // 32) ** 2, 2 * (res // 16) ** 2           # tokens at level 2 / level 1, CFG batch 2
shapes = [("l2 qkv", T2, 3840, 1280, 60), ("l2 to_out", T2, 1280, 1280, 120), ("l2 cross q", T2, 1280, 1280, 60),
          ("l2 ff2", T2, 1280, 5120, 60), ("l2 ff1 (8C)", T2, 10240, 1280, 60),
          ("l1 qkv", T1, 1920, 640, 10), ("l1 to_out", T1, 640, 640, 20), ("l1 ff2", T1, 640, 2560, 10), ("l1 ff1 (8C)", T1, 5120, 640, 10),
          ("text kv l2", 154, 2560, 2048, 60)]
print(f"== Linear shapes of one SDXL {res}^2 step (M = tokens of the CFG pair), fp16")
tot_ours = tot_lib = 0.0
for name, M, N, K, count in shapes:
    sets = [((torch.randn(M, K, device="cuda").half()), (torch.randn(N, K, device="cuda") / K ** 0.5).half(),
             torch.randn(N, device="cuda").half()) for _ in range(NSETS)]
    t_lib = timeit(lambda s_: (lambda: F.linear(*s_)), sets)
    t_ours = timeit(lambda s_: (lambda: ops.linear(*s_)), sets)
    del sets
    fl = 2.0 * M * N * K
    tot_ours += t_ours * count; tot_lib += t_lib * count
    print(f"{name:14s} M={M:6d} N={N:6d} K={K:5d} x{count:3d}: ours {t_ours * 1e3:8.1f} us {fl / t_ours / 1e9:7.1f} TFLOP/s | "
          f"cuBLAS {t_lib * 1e3:8.1f} us {fl / t_lib / 1e9:7.1f} TFLOP/s | x{t_lib / t_ours:.2f}")
print(f"   per-step total: ours {tot_ours:.3f} ms | cuBLAS {tot_lib:.3f} ms")
print("== GEGLU projection: fused (one kernel) vs F.linear + df_geglu (two kernels)")
for name, M, K, D, count in [("l2 ff1+geglu", T2, 1280, 5120, 60), ("l1 ff1+geglu", T1, 640, 2560, 10)]:
    sets = []
    for _ in range(NSETS):
        x = torch.randn(M, K, device="cuda").half()
        w = (torch.randn(2 * D, K, device="cuda") / K ** 0.5).half()
        bias = torch.randn(2 * D, device="cuda").half()
        blk = ops.geglu_block(M, 2 * D, K)
        sets.append((x, w, bias) + ops.geglu_interleave(w, bias, blk) + (blk,))
    t_two = timeit(lambda s_: (lambda: ops.geglu(F.linear(s_[0], s_[1], s_[2]))), sets)
    t_one = timeit(lambda s_: (lambda: ops.linear_geglu(s_[0], s_[3], s_[4], s_[5])), sets)
    del sets
    fl = 2.0 * M * 2 * D * K
    print(f"{name:14s} M={M:6d} K={K:5d} D={D:5d} blk={blk} x{count:3d}: fused {t_one * 1e3:8.1f} us {fl / t_one / 1e9:7.1f} TFLOP/s | "
          f"cuBLAS+geglu {t_two * 1e3:8.1f} us | x{t_two / t_one:.2f}   (saves {(t_two - t_one) * count:.3f} ms/step)")
