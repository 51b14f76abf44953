"""Multi-rank driver of the PRODUCT naive-patch path (parallelism="naive_patch") for the GPU tests (test infrastructure).

Same process layout as mp_product.py: one process per rank, gloo for the rendezvous only, the final epsilon gather through the
CUDA peer-memory kernels; with fewer GPUs than ranks the ranks share cuda:0 (DISTRIFUSER_B200_SHARE_GPU=1)."""
from __future__ import annotations

import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _setup(rank, case, port, use_graph):
    """-> (pipeline, seeded-weights unet config) of this rank, built through the public API."""
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
    cfg = DistriConfig(height=8 * case.latent, width=8 * case.latent, do_classifier_free_guidance=case.cfg,
                       split_batch=case.split_batch, use_cuda_graph=use_graph, parallelism="naive_patch",
                       split_scheme=case.scheme)
    ucfg = W.unet_config(case.family)
    unet = UNet2DConditionModel(**ucfg)
    unet.load_state_dict(W.make_unet(case.family, case.weight_seed).state_dict(), strict=True)   # the golden run's weights
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


def _unet_worker(rank, case, port, outdir, use_graph):
    from oracle import workloads as W
    pipe, ucfg = _setup(rank, case, port, use_graph)
    model, dev = pipe.pipeline.unet, pipe.distri_config.device
    outs = []
    with torch.no_grad():
        model.set_counter(0)                                               # pipelines.py:57
        for t in range(case.steps):
            inp = W.unet_inputs(case, t, ucfg)
            half = lambda x: x.to(dev, torch.float16)
            kw = dict(sample=half(inp["sample"]), timestep=inp["timestep"].to(dev).float(),
                      encoder_hidden_states=half(inp["encoder_hidden_states"]))
            if inp["added_cond_kwargs"] is not None:
                kw["added_cond_kwargs"] = {k: half(v) for k, v in inp["added_cond_kwargs"].items()}
            outs.append(model(**kw, return_dict=False)[0].float().cpu().clone())
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    _finish(pipe, case.world_size)


def _traj_worker(rank, case, port, outdir, num_steps, guidance, use_graph):
    pipe, _ = _setup(rank, case, port, use_graph)
    run = lambda: pipe(prompt="a photo", num_inference_steps=num_steps, guidance_scale=guidance,
                       generator=torch.Generator().manual_seed(case.input_seed)).images      # public API
    lat = run()
    lat2 = run()
    torch.cuda.synchronize()
    assert torch.equal(lat, lat2), "second image with the same seed differs from the first"
    torch.save(lat.float().cpu(), os.path.join(outdir, f"rank{rank}.pt"))
    _finish(pipe, case.world_size)


def _run(worker, case, *args):
    from oracle.harness import free_port
    from torch import multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        if case.world_size == 1:
            worker(0, case, 0, d, *args)
        else:
            mp.spawn(worker, args=(case, free_port(), d, *args), nprocs=case.world_size, join=True)
        return [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(case.world_size)]


def run_naive_product_unet(case, use_graph=False):
    """-> per rank, the eps prediction of each of case.steps UNet calls (counter 0, 1, ...)."""
    return _run(_unet_worker, case, use_graph)


def run_naive_product_trajectory(case, num_steps=8, guidance=5.0, use_graph=True):
    """-> per rank, the final latents of the pipeline (a second image with the same seed is asserted bit-identical)."""
    return _run(_traj_worker, case, num_steps, guidance, use_graph)
