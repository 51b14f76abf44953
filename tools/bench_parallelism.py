#!/usr/bin/env python
"""ms/image of displaced patch parallelism (parallelism="patch") against the naive patch baseline (parallelism="naive_patch",
split_scheme row / col / alternate) on bench.py's workload: synthetic SDXL UNet (random weights, seed 0), 50 Euler steps,
CFG (guidance 5), CUDA graphs, latents and prompt embeddings resident on the device.  One pipeline per configuration is
built up front; the timed rounds then alternate the configurations, so drift of the card (clocks, power, neighbours) falls
on all of them alike.  Prints one JSON line with the card name and power limit beside the numbers.

    python -m torch.distributed.run --nproc-per-node N tools/bench_parallelism.py [--rounds 3] [--images 2] [--resolution 1024]
        [--dump-outputs DIR]      # rank 0 writes each configuration's final latents to DIR/<config>.npy

Any N from 1 to 8.  An odd N runs both CFG branches on every rank (split_batch=False: two CFG groups need an even N); an even
N splits the CFG batch unless --no-split-batch.  Naive patch needs strips of whole latent rows / columns: a configuration
that does not cut into them at the chosen resolution is skipped and the reason recorded.  At --resolution 1536 (192 latent
rows, 48 SDXL row units) every configuration runs at N in {1, 2, 3, 4, 6, 8}; at 1024 naive patch runs at N in {1, 2, 4, 8}
only, and at N = 5 or 7 only patch parallelism runs at either resolution.

One GPU per rank: with fewer GPUs than ranks the ranks would time-slice one device, so the script then times nothing and
reports "not measured"."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CONFIGS = (("patch", "row"), ("naive_patch", "row"), ("naive_patch", "col"), ("naive_patch", "alternate"))


def card() -> dict:
    """Name and power limit of this rank's GPU (read-only query)."""
    import torch
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        idx = torch.cuda.current_device()
        r = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = [f.strip() for f in r.stdout.strip().split(",")[:2]]
        info["power_limit_w"], info["sm_max_mhz"] = float(pl), float(mx)
    except Exception as e:                                           # the numbers stay, labelled without a power limit
        info["power_limit_error"] = repr(e)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=2, help="images per configuration and round")
    ap.add_argument("--warmup", type=int, default=2, help="untimed images per configuration")
    ap.add_argument("--resolution", type=int, default=1024)
    ap.add_argument("--no-split-batch", action="store_true", help="every rank runs both CFG branches on its patch")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    a = ap.parse_args()

    import torch
    from torch import distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if ngpu < world:
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps({"bench": "parallelism", "world_size": world, "gpus": ngpu,
                              "result": f"not measured: {world} ranks need {world} GPUs, this box has {ngpu}"}), flush=True)
        return

    import bench
    from distrifuser_b200.pipelines import DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig

    R = a.resolution
    split = not a.no_split_batch and world % 2 == 0
    pipes, skipped = {}, {}
    for par, scheme in CONFIGS:
        name = par if par == "patch" else f"naive_{scheme}"
        try:
            cfg = DistriConfig(height=R, width=R, split_batch=split, parallelism=par, split_scheme=scheme)
        except ValueError as e:                                      # naive strips that are not whole latent rows / columns
            if par != "naive_patch":
                raise
            skipped[name] = str(e)
            continue
        pipe = DistriSDXLPipeline.from_synthetic(cfg, seed=0)
        pipe.set_progress_bar_config(disable=True)
        pipes[name] = pipe
    cfg = next(iter(pipes.values())).distri_config
    rank, dev = cfg.rank, cfg.device
    io = bench.make_inputs(argparse.Namespace(model="sdxl"), next(iter(pipes.values())), dev, R)

    def image(pipe):
        return pipe(prompt_embeds=io["embeds_d"], pooled_prompt_embeds=io["pooled_d"], latents=io["lat_d"],
                    num_inference_steps=bench.STEPS_PER_IMAGE, guidance_scale=5.0, output_type="latent")

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    last = {}
    for name, pipe in pipes.items():
        for _ in range(a.warmup):
            last[name] = image(pipe).images.float().cpu()
    times = {name: [] for name in pipes}
    for _ in range(a.rounds):
        for name, pipe in pipes.items():
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.images):
                image(pipe)
            e1.record()
            barrier()
            ms = torch.tensor([e0.elapsed_time(e1) / a.images], device=dev)
            if world > 1:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            times[name].append(ms.item())
    if a.dump_outputs and rank == 0:
        bench.dump_outputs(a.dump_outputs, last)
    gpu = card()
    if rank == 0:
        print(json.dumps({
            "bench": "parallelism", "workload": f"synthetic SDXL {R}x{R}, {bench.STEPS_PER_IMAGE} Euler steps, CFG, CUDA graphs",
            "world_size": world, "split_batch": split, "card": gpu,
            "ms_per_image": {k: round(statistics.median(v), 1) for k, v in times.items()},
            "ms_per_image_rounds": {k: [round(x, 1) for x in v] for k, v in times.items()},
            "skipped": skipped,
        }), flush=True)
    barrier()
    for pipe in pipes.values():
        if pipe.comm_manager is not None:
            pipe.comm_manager.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
