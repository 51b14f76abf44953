"""Summarises an `ncu --metrics gpu__time_duration.sum --csv` launch list: time share per kernel family."""
import csv
import re
import sys
from collections import defaultdict


def family(name: str) -> str:
    n = name
    for pat, fam in ((r"fmha_fwd_kernel", "OURS fmha_fwd_kernel (wgmma)"), (r"gn_fused_kernel", "OURS gn_fused_kernel"),
                     (r"halo_|publish_kernel|wait_kernel|step_begin|out_scatter|out_collect", "OURS comm/halo kernels"),
                     (r"geglu_kernel", "OURS geglu_kernel"), (r"add_layernorm_kernel", "OURS add_layernorm_kernel"),
                     (r"bias_residual_add_kernel", "OURS bias_residual_add_kernel (conv bias + residual)"),
                     (r"linear_kernel|gemm_kernel", "OURS wgmma GEMM (df_linear)"),
                     # cuDNN's sm100 convs are "cutlass3x_sm100 ... fprop / implicit gemm" kernels: match them BEFORE the GEMM row
                     (r"cudnn|conv|implicit|fprop|wgrad|dgrad|nhwc|nchw", "library conv (cuDNN)"),
                     (r"nvjet|cutlass.*gemm|sm\d+_xmma_gemm|cublas|gemm|gemv", "library GEMM (cuBLAS)"),
                     (r"layer_norm|LayerNorm", "torch layer_norm"), (r"gelu|GeluCUDAKernel", "torch gelu"),
                     (r"elementwise|vectorized|CatArray|copy|upsample|fill", "torch elementwise / copy / cat")):
        if re.search(pat, n, re.I):
            return fam
    return "other: " + n[:60]


def main(path):
    rows = list(csv.reader(l for l in open(path, errors="ignore") if l.startswith('"')))
    hdr = rows[0]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg, cnt, total = defaultdict(float), defaultdict(int), 0.0
    for r in rows[1:]:
        if len(r) <= vi:
            continue
        v = float(r[vi].replace(",", ""))
        v = v / 1e3 if r[ui] in ("ns", "nsecond") else (v if r[ui] in ("us", "usecond") else v * 1e3)
        f = family(r[ki])
        agg[f] += v
        cnt[f] += 1
        total += v
    print(f"total kernel time {total / 1e3:.3f} ms over {sum(cnt.values())} launches (ncu: serialised, cold-cache; compare shares)")
    for f, v in sorted(agg.items(), key=lambda kv: -kv[1]):
        print(f"{v / 1e3:9.3f} ms  {100 * v / total:5.1f}%  {cnt[f]:5d} launches  {f}")


if __name__ == "__main__":
    main(sys.argv[1])
