#!/usr/bin/env python
"""ms/image of bench.py's workload with and without a ControlNet: synthetic SDXL UNet (random weights, seed 0), 50 Euler steps,
CFG (guidance 5), CUDA graphs, patch parallelism, latents and prompt embeddings resident on the device.  The ControlNet is
`ControlNetModel.from_unet` with its zero-initialised layers drawn at random (a trained ControlNet's are not zero), and a random
conditioning image.  Both pipelines are built up front and the timed rounds alternate them, so drift of the card falls on both
alike.  Prints one JSON line with the card name and power limit beside the numbers.

    python tools/bench_controlnet.py --gpus 1 [--rounds 3] [--images 2] [--resolution 1024]
    python -m torch.distributed.run --nproc-per-node N tools/bench_controlnet.py [...]

One GPU per rank: with fewer GPUs than ranks nothing is timed and the result says "not measured"."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=None, help="expected rank count (default: WORLD_SIZE, or 1)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=2, help="images per configuration and round")
    ap.add_argument("--warmup", type=int, default=1, help="untimed images per configuration")
    ap.add_argument("--resolution", type=int, default=1024)
    a = ap.parse_args()

    import torch
    from torch import distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if a.gpus is not None and a.gpus != world:
        raise SystemExit(f"--gpus {a.gpus} but {world} ranks: run N > 1 under torch.distributed.run --nproc-per-node N")
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if ngpu < world or ngpu == 0:
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps({"bench": "controlnet", "world_size": world, "gpus": ngpu,
                              "result": f"not measured: {world} ranks need {world} GPUs, this box has {ngpu}"}), flush=True)
        return

    import bench
    from bench_parallelism import card
    from distrifuser_b200.compat.controlnet import ControlNetModel
    from distrifuser_b200.compat.unet_2d_condition import SDXL, UNet2DConditionModel
    from distrifuser_b200.pipelines import DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig

    R = a.resolution
    split = world % 2 == 0
    pipes = {}
    for name in ("unet", "unet+controlnet"):
        cfg = DistriConfig(height=R, width=R, split_batch=split)
        torch.manual_seed(0)
        with torch.device(cfg.device):
            unet = UNet2DConditionModel(**SDXL)
        cn = None
        if name != "unet":
            cn = ControlNetModel.from_unet(unet)
            g = torch.Generator(device=cfg.device).manual_seed(1)
            with torch.no_grad():
                for conv in [cn.controlnet_cond_embedding.conv_out, *cn.zero_convs()]:
                    conv.weight.copy_(torch.randn(conv.weight.shape, generator=g, device=cfg.device) * 0.02)
                    conv.bias.zero_()
        pipe = DistriSDXLPipeline.from_synthetic(cfg, unet=unet, controlnet=cn)
        pipe.set_progress_bar_config(disable=True)
        pipes[name] = pipe
    cfg = pipes["unet"].distri_config
    rank, dev = cfg.rank, cfg.device
    io = bench.make_inputs(argparse.Namespace(model="sdxl"), pipes["unet"], dev, R)
    cond = torch.rand((1, 3, R, R), generator=torch.Generator(device=dev).manual_seed(2), device=dev) * 2 - 1

    def image(name):
        kw = dict(image=cond, controlnet_conditioning_scale=1.0) if name != "unet" else {}
        return pipes[name](prompt_embeds=io["embeds_d"], pooled_prompt_embeds=io["pooled_d"], latents=io["lat_d"],
                           num_inference_steps=bench.STEPS_PER_IMAGE, guidance_scale=5.0, output_type="latent", **kw)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for name in pipes:
        for _ in range(a.warmup):
            image(name)
    times = {name: [] for name in pipes}
    for _ in range(a.rounds):
        for name in pipes:
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.images):
                image(name)
            e1.record()
            barrier()
            ms = torch.tensor([e0.elapsed_time(e1) / a.images], device=dev)
            if world > 1:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            times[name].append(ms.item())
    gpu = card()
    if rank == 0:
        med = {k: round(statistics.median(v), 1) for k, v in times.items()}
        print(json.dumps({
            "bench": "controlnet", "workload": f"synthetic SDXL {R}x{R}, {bench.STEPS_PER_IMAGE} Euler steps, CFG, CUDA graphs",
            "world_size": world, "split_batch": split, "card": gpu, "ms_per_image": med,
            "ms_per_image_rounds": {k: [round(x, 1) for x in v] for k, v in times.items()},
            "controlnet_overhead": round(med["unet+controlnet"] / med["unet"] - 1, 3),
        }), flush=True)
    barrier()
    for pipe in pipes.values():
        if pipe.comm_manager is not None:
            pipe.comm_manager.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
