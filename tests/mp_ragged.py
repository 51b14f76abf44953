"""Multi-rank drivers for patch parallelism on uneven row strips (test infrastructure): the CPU oracle extended to uneven
strips (tests/ragged_oracle.py, fp32, gloo) and the
product path (fp16, sm_90a kernels, peer memory) on the same seeded tiny UNet at a latent of H x W, where the patch count
need not divide the latent height into equal strips.  oracle/harness.py and mp_product.py drive square latents only."""
from __future__ import annotations

import dataclasses
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


@dataclasses.dataclass(frozen=True)
class RaggedCase:
    name: str
    family: str = "tiny_sdxl"
    world_size: int = 2
    cfg: bool = True
    split_batch: bool = False
    mode: str = "corrected_async_gn"
    warmup_steps: int = 1
    steps: int = 4
    lat_h: int = 36                  # latent rows (image height / 8)
    lat_w: int = 28
    comm_checkpoint: int = 20
    weight_seed: int = 0
    input_seed: int = 4321

    @property
    def batch(self):
        return 2 if self.cfg else 1


def unet_inputs(case: RaggedCase, step: int, ucfg: dict):
    """Inputs of denoise call `step` at a [B, 4, lat_h, lat_w] latent (oracle.workloads.unet_inputs, non-square)."""
    g = torch.Generator().manual_seed(case.input_seed + 7919 * step)
    B = case.batch
    sample = torch.randn(B, 4, case.lat_h, case.lat_w, generator=g)
    g2 = torch.Generator().manual_seed(case.input_seed)
    ehs = torch.randn(B, 77, ucfg["cross_attention_dim"], generator=g2)
    timestep = torch.full((B,), 981 - 20 * step, dtype=torch.long)
    added = None
    if ucfg.get("addition_embed_type") == "text_time":
        pooled = ucfg["projection_class_embeddings_input_dim"] - 6 * ucfg["addition_time_embed_dim"]
        H, W = float(8 * case.lat_h), float(8 * case.lat_w)
        added = {"text_embeds": torch.randn(B, pooled, generator=g2), "time_ids": torch.tensor([[H, W, 0.0, 0.0, H, W]] * B)}
    return dict(sample=sample, timestep=timestep, encoder_hidden_states=ehs, added_cond_kwargs=added)


def _spawn(fn, world, args):
    from oracle.harness import free_port
    from torch import multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        if world == 1:
            fn(0, *args, 0, d)
        else:
            mp.spawn(fn, args=(*args, free_port(), d), nprocs=world, join=True)
        return [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(world)]


# ------------------------------------------------------------------------------------------------------------ oracle (CPU)
def _oracle_worker(rank, case, bessel, port, outdir):
    from oracle import harness as Hn
    from ragged_oracle import RaggedUNetPP
    from oracle import workloads as W
    Hn._paths("oracle")
    Hn._init(rank, case.world_size, port)
    cfg = W.DuckConfig(case.world_size, rank, height=8 * case.lat_h, width=8 * case.lat_w, do_classifier_free_guidance=case.cfg,
                       split_batch=case.split_batch, warmup_steps=case.warmup_steps, comm_checkpoint=case.comm_checkpoint,
                       mode=case.mode)
    if case.world_size > 1:
        Hn._groups(cfg)
    ucfg = W.unet_config(case.family)
    model = RaggedUNetPP(W.make_unet(case.family, case.weight_seed), cfg, bessel=bessel)
    outs = []
    with torch.no_grad():
        model.prepare(unet_inputs(case, 0, ucfg))
        model.set_counter(0)
        for t in range(case.steps):
            outs.append(model(**unet_inputs(case, t, ucfg)).clone())
    torch.save((outs, model.units), os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


def run_oracle_unet(case: RaggedCase, bessel: bool = True):
    """-> (outs[step] = eps [B, 4, lat_h, lat_w], the row plan's units); every rank's output must be identical."""
    per_rank = _spawn(_oracle_worker, case.world_size, (case, bessel))
    for outs, _ in per_rank[1:]:
        for a, b in zip(per_rank[0][0], outs):
            assert torch.equal(a, b), "final output must be identical on all ranks"
    return per_rank[0][0], per_rank[0][1]


def _oracle_traj_worker(rank, case, num_steps, guidance, port, outdir):
    from oracle import harness as Hn
    from ragged_oracle import RaggedUNetPP
    from oracle import workloads as W
    Hn._paths("oracle")
    from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline
    Hn._init(rank, case.world_size, port)
    cfg = W.DuckConfig(case.world_size, rank, height=8 * case.lat_h, width=8 * case.lat_w, do_classifier_free_guidance=case.cfg,
                       split_batch=case.split_batch, warmup_steps=case.warmup_steps, comm_checkpoint=case.comm_checkpoint,
                       mode=case.mode)
    if case.world_size > 1:
        Hn._groups(cfg)
    ucfg = W.unet_config(case.family)
    unet = W.make_unet(case.family, case.weight_seed)
    model = RaggedUNetPP(unet, cfg)
    model.prepare(unet_inputs(case, 0, ucfg))
    pipe = SyntheticLatentPipeline(Hn._OracleUNetAdapter(model, unet.config), sdxl=ucfg.get("addition_embed_type") == "text_time",
                                   device="cpu", dtype=torch.float32)
    model.set_counter(0)
    g = torch.Generator().manual_seed(case.input_seed)
    with torch.no_grad():
        lat = pipe(prompt="a photo", height=8 * case.lat_h, width=8 * case.lat_w, num_inference_steps=num_steps,
                   guidance_scale=guidance, generator=g).images
    torch.save(lat, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


def run_oracle_trajectory(case: RaggedCase, num_steps=8, guidance=5.0):
    outs = _spawn(_oracle_traj_worker, case.world_size, (case, num_steps, guidance))
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    return outs[0]


# ------------------------------------------------------------------------------------------------------------ product (GPU)
def _setup_product(rank, case, port, use_graph):
    from torch import distributed as dist
    if case.world_size > 1:
        if torch.cuda.device_count() < case.world_size:
            os.environ["DISTRIFUSER_B200_SHARE_GPU"] = "1"
        os.environ["LOCAL_RANK"] = str(rank)
        dist.init_process_group("gloo", rank=rank, world_size=case.world_size, init_method=f"tcp://127.0.0.1:{port}")
    from oracle import workloads as W
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(height=8 * case.lat_h, width=8 * case.lat_w, do_classifier_free_guidance=case.cfg,
                       split_batch=case.split_batch, warmup_steps=case.warmup_steps, mode=case.mode, use_cuda_graph=use_graph)
    ucfg = W.unet_config(case.family)
    unet = UNet2DConditionModel(**ucfg)
    unet.load_state_dict(W.make_unet(case.family, case.weight_seed).state_dict(), strict=True)
    cls = DistriSDXLPipeline if ucfg.get("addition_embed_type") == "text_time" else DistriSDPipeline
    return cfg, ucfg, cls.from_synthetic(cfg, unet=unet)


def _teardown(case, pipe):
    from torch import distributed as dist
    if case.world_size > 1:
        dist.barrier()
        if pipe.comm_manager is not None:
            pipe.comm_manager.close()
        dist.destroy_process_group()


def _product_worker(rank, case, use_graph, port, outdir):
    cfg, ucfg, pipe = _setup_product(rank, case, port, use_graph)
    model = pipe.pipeline.unet
    outs = []
    with torch.no_grad():
        model.set_counter(0)
        for t in range(case.steps):
            inp = unet_inputs(case, t, ucfg)
            dev = lambda x: x.to(cfg.device, torch.float16) if x.is_floating_point() else x.to(cfg.device)
            kw = dict(sample=dev(inp["sample"]), timestep=inp["timestep"].to(cfg.device).float(),
                      encoder_hidden_states=dev(inp["encoder_hidden_states"]))
            if inp["added_cond_kwargs"] is not None:
                kw["added_cond_kwargs"] = {k: dev(v) for k, v in inp["added_cond_kwargs"].items()}
            outs.append(model(**kw, return_dict=False)[0].float().cpu().clone())
    torch.cuda.synchronize()
    torch.save((outs, model.row_units), os.path.join(outdir, f"rank{rank}.pt"))
    _teardown(case, pipe)


def run_product_unet(case: RaggedCase, use_graph=False):
    """-> per rank: (outs[step], row units of the plan)."""
    return _spawn(_product_worker, case.world_size, (case, use_graph))


def _product_traj_worker(rank, case, num_steps, guidance, port, outdir):
    cfg, ucfg, pipe = _setup_product(rank, case, port, True)
    g = torch.Generator().manual_seed(case.input_seed)
    lat = pipe(prompt="a photo", num_inference_steps=num_steps, guidance_scale=guidance, generator=g).images
    g2 = torch.Generator().manual_seed(case.input_seed)
    lat2 = pipe(prompt="a photo", num_inference_steps=num_steps, guidance_scale=guidance, generator=g2).images
    torch.cuda.synchronize()
    assert torch.equal(lat, lat2), "second image with the same seed differs from the first"
    torch.save(lat.float().cpu(), os.path.join(outdir, f"rank{rank}.pt"))
    _teardown(case, pipe)


def run_product_trajectory(case: RaggedCase, num_steps=8, guidance=5.0):
    return _spawn(_product_traj_worker, case.world_size, (case, num_steps, guidance))
