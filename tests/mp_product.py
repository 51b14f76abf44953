"""Multi-rank driver of the PRODUCT path for the parity tests and multi-GPU runs (test infrastructure).

One process per rank; gloo is only the rendezvous plane (IPC-handle exchange + barriers), every activation moves
through the CUDA peer-memory kernels.  With fewer GPUs than ranks the ranks share cuda:0
(DISTRIFUSER_B200_SHARE_GPU=1): CUDA IPC works between processes on one device, so a 1-GPU box still exercises
the multi-rank slots / flags / epochs (slowly: spin-waits are time-sliced)."""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _setup(rank, case, port, use_graph):
    """-> this rank's pipeline, built through the public API around the golden run's seeded weights, and the UNet config."""
    from torch import distributed as dist
    world = case.world_size
    if world > 1:
        if torch.cuda.device_count() < world:
            os.environ["DISTRIFUSER_B200_SHARE_GPU"] = "1"
        os.environ["LOCAL_RANK"] = str(rank)
        dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    from oracle import workloads as W
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(**case.config_kwargs(), use_cuda_graph=use_graph)
    ucfg = W.unet_config(case.family)
    unet = UNet2DConditionModel(**ucfg)
    unet.load_state_dict(W.make_unet(case.family, case.weight_seed).state_dict(), strict=True)
    cls = DistriSDXLPipeline if ucfg.get("addition_embed_type") == "text_time" else DistriSDPipeline
    return cls.from_synthetic(cfg, unet=unet), ucfg


def _finish(pipe, world):
    from torch import distributed as dist
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        if pipe.comm_manager is not None:
            pipe.comm_manager.close()
        dist.destroy_process_group()


def _unet_worker(rank, case, use_graph, row_units, port, outdir):
    from oracle import workloads as W
    pipe, ucfg = _setup(rank, case, port, use_graph)
    model, dev = pipe.pipeline.unet, pipe.distri_config.device
    if row_units is not None:
        assert model.row_units == row_units, f"rank {rank}: row plan {model.row_units}, expected {row_units}"
    outs = []
    with torch.no_grad():
        model.set_counter(0)                                               # pipelines.py:57
        for t in range(case.steps):
            inp = W.unet_inputs(case, t, ucfg)
            to_dev = lambda x: x.to(dev, torch.float16) if x.is_floating_point() else x.to(dev)
            kw = dict(sample=to_dev(inp["sample"]), timestep=inp["timestep"].to(dev).float(),
                      encoder_hidden_states=to_dev(inp["encoder_hidden_states"]))
            if inp["added_cond_kwargs"] is not None:
                kw["added_cond_kwargs"] = {k: to_dev(v) for k, v in inp["added_cond_kwargs"].items()}
            outs.append(model(**kw, return_dict=False)[0].float().cpu().clone())
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    _finish(pipe, case.world_size)


def _traj_worker(rank, case, num_steps, guidance, use_graph, port, outdir):
    pipe, _ = _setup(rank, case, port, use_graph)
    run = lambda: pipe(prompt="a photo", num_inference_steps=num_steps, guidance_scale=guidance,
                       generator=torch.Generator().manual_seed(case.input_seed)).images      # public API
    lat = run()
    # a second image with the same seed must reproduce the first bit for bit: nothing (epoch banks, text-KV cache, stale
    # activations, graph state) may leak from one image into the next (pipelines.py:57 resets the counters)
    lat2 = run()
    torch.cuda.synchronize()
    assert torch.equal(lat, lat2), "second image with the same seed differs from the first"
    torch.save(lat.float().cpu(), os.path.join(outdir, f"rank{rank}.pt"))
    _finish(pipe, case.world_size)


def run_product_unet(case, use_graph=False, row_units=None):
    """-> per rank, the eps prediction of each of case.steps UNet calls (counter 0, 1, ...).  The case picks the
    parallelism (UNetCase, RaggedCase: patch; NaiveCase: naive patch); `row_units`, when given, is asserted to be every rank's
    row plan."""
    from oracle.harness import run_ranks
    return run_ranks(_unet_worker, case, use_graph, row_units)


def run_product_trajectory(case, num_steps=8, guidance=5.0, use_graph=True):
    """-> per rank, the final latents of the pipeline (a second image with the same seed is asserted bit-identical)."""
    from oracle.harness import run_ranks
    return run_ranks(_traj_worker, case, num_steps, guidance, use_graph)
