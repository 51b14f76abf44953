"""Multi-rank driver of the PRODUCT path for the parity tests and multi-GPU runs (test infrastructure).

One process per rank; gloo is only the rendezvous plane (IPC-handle exchange + barriers), every activation moves
through the CUDA peer-memory kernels.  With fewer GPUs than ranks the ranks share cuda:0
(DISTRIFUSER_B200_SHARE_GPU=1): CUDA IPC works between processes on one device, so a 1-GPU box still exercises
the multi-rank slots / flags / epochs (slowly: spin-waits are time-sliced).

`controlnet` spells the ControlNet as oracle.harness.run_unet does: None (none), "drawn" (seeded, its zero-initialised layers
drawn) or "zero" (as initialised); the product loads the oracle's seeded weights strict=True."""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _init(rank, case, port):
    from torch import distributed as dist
    world = case.world_size
    if world > 1:
        if torch.cuda.device_count() < world:
            os.environ["DISTRIFUSER_B200_SHARE_GPU"] = "1"
        os.environ["LOCAL_RANK"] = str(rank)
        dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")


def _pipeline(case, use_graph, controlnet=None):
    """-> this rank's pipeline, built through the public API around the golden run's seeded weights."""
    from oracle import workloads as W
    from distrifuser_b200.compat.controlnet import ControlNetModel
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(**case.config_kwargs(), use_cuda_graph=use_graph)
    ucfg = W.unet_config(case.family)
    unet = UNet2DConditionModel(**ucfg)
    unet.load_state_dict(W.make_unet(case.family, case.weight_seed).state_dict(), strict=True)
    cn = None
    if controlnet is not None:
        cn = ControlNetModel(**ucfg)
        cn.load_state_dict(W.make_controlnet(case.family, case.weight_seed, zero=controlnet == "zero").state_dict(),
                           strict=True)
    cls = DistriSDXLPipeline if ucfg.get("addition_embed_type") == "text_time" else DistriSDPipeline
    return cls.from_synthetic(cfg, unet=unet, controlnet=cn)


def _unet_steps(pipe, case, controlnet=None, scale=1.0):
    """-> the eps prediction of each of case.steps UNet calls (counter 0, 1, ...); `scale`: a float, or one per step."""
    from oracle import workloads as W
    model, dev = pipe.pipeline.unet, pipe.distri_config.device
    ucfg = W.unet_config(case.family)
    to_dev = lambda x: x.to(dev, torch.float16) if x.is_floating_point() else x.to(dev)
    cond = to_dev(W.cond_image(case)).expand(case.batch, -1, -1, -1)
    outs = []
    with torch.no_grad():
        model.set_counter(0)                                               # pipelines.py:57
        for t in range(case.steps):
            inp = W.unet_inputs(case, t, ucfg)
            kw = dict(sample=to_dev(inp["sample"]), timestep=inp["timestep"].to(dev).float(),
                      encoder_hidden_states=to_dev(inp["encoder_hidden_states"]))
            if inp["added_cond_kwargs"] is not None:
                kw["added_cond_kwargs"] = {k: to_dev(v) for k, v in inp["added_cond_kwargs"].items()}
            if controlnet is not None:
                kw.update(controlnet_cond=cond, conditioning_scale=scale[t] if isinstance(scale, (list, tuple)) else scale)
            outs.append(model(**kw, return_dict=False)[0].float().cpu().clone())
    return outs


def _finish(pipes, world):
    from torch import distributed as dist
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        for pipe in pipes:
            if pipe.comm_manager is not None:
                pipe.comm_manager.close()
        dist.destroy_process_group()


def _unet_worker(rank, case, use_graph, row_units, controlnet, scale, port, outdir):
    _init(rank, case, port)
    pipe = _pipeline(case, use_graph, controlnet)
    if row_units is not None:
        units = pipe.pipeline.unet.row_units
        assert units == row_units, f"rank {rank}: row plan {units}, expected {row_units}"
    torch.save(_unet_steps(pipe, case, controlnet, scale), os.path.join(outdir, f"rank{rank}.pt"))
    _finish([pipe], case.world_size)


def _zero_premise_worker(rank, case, port, outdir):
    """Both pipelines in ONE process, so that cuDNN's autotuned algorithms are the same for both."""
    _init(rank, case, port)
    plain, zero = _pipeline(case, True), _pipeline(case, True, "zero")
    torch.save((_unet_steps(plain, case), _unet_steps(zero, case, "zero")), os.path.join(outdir, f"rank{rank}.pt"))
    _finish([plain, zero], case.world_size)


def _traj_worker(rank, case, num_steps, guidance, use_graph, controlnet, port, outdir):
    from oracle import workloads as W
    _init(rank, case, port)
    pipe = _pipeline(case, use_graph, controlnet)
    cn_kw = {} if controlnet is None else dict(image=W.cond_image(case), controlnet_conditioning_scale=1.0)
    run = lambda: pipe(prompt="a photo", num_inference_steps=num_steps, guidance_scale=guidance,
                       generator=torch.Generator().manual_seed(case.input_seed), **cn_kw).images     # public API
    lat = run()
    # a second image with the same seed must reproduce the first bit for bit: nothing (epoch banks, text-KV cache, stale
    # activations, graph state) may leak from one image into the next (pipelines.py:57 resets the counters)
    lat2 = run()
    torch.cuda.synchronize()
    assert torch.equal(lat, lat2), "second image with the same seed differs from the first"
    torch.save(lat.float().cpu(), os.path.join(outdir, f"rank{rank}.pt"))
    _finish([pipe], case.world_size)


def run_product_unet(case, use_graph=False, row_units=None, controlnet=None, scale=1.0):
    """-> per rank, the eps prediction of each of case.steps UNet calls (counter 0, 1, ...).  The case picks the
    parallelism (UNetCase, RaggedCase: patch; NaiveCase: naive patch); `row_units`, when given, is asserted to be every rank's
    row plan.  With `controlnet`, each call takes the case's conditioning image at conditioning scale `scale` (a float, or
    one per step)."""
    from oracle.harness import run_ranks
    return run_ranks(_unet_worker, case, use_graph, row_units, controlnet, scale)


def run_zero_premise(case):
    """-> per rank, (outputs without a ControlNet, outputs with a zero-initialised one), CUDA graphs on."""
    from oracle.harness import run_ranks
    return run_ranks(_zero_premise_worker, case)


def run_product_trajectory(case, num_steps=8, guidance=5.0, use_graph=True, controlnet=None):
    """-> per rank, the final latents of the pipeline (a second image with the same seed is asserted bit-identical).  With
    `controlnet`, the pipeline takes the case's conditioning image at scale 1."""
    from oracle.harness import run_ranks
    return run_ranks(_traj_worker, case, num_steps, guidance, use_graph, controlnet)
