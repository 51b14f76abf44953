"""Profiling driver: builds the synthetic SDXL pipeline (eager, no CUDA graph) and brackets ONE asynchronous denoise
step with cudaProfilerStart/Stop so that `ncu --profile-from-start off` lists exactly the kernels of one step.

  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file launches.csv \
      python tools/profile_step.py --resolution 1024
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, default=1024)
    ap.add_argument("--model", default="sdxl")
    ap.add_argument("--warm", type=int, default=6, help="un-profiled UNet calls before the profiled one (>= warmup_steps+2)")
    a = ap.parse_args()
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(height=a.resolution, width=a.resolution, use_cuda_graph=False)
    cls = DistriSDXLPipeline if a.model == "sdxl" else DistriSDPipeline
    pipe = cls.from_synthetic(cfg, seed=0)
    unet, si = pipe.pipeline.unet, pipe.static_inputs
    unet.set_counter(0)
    with torch.no_grad():
        for _ in range(a.warm):
            unet(**si, return_dict=False)
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        unet(**si, return_dict=False)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
    print("profiled one denoise step", flush=True)


if __name__ == "__main__":
    main()
