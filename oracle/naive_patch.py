"""TEST INFRASTRUCTURE (oracle) -- the naive patch baseline (parallelism="naive_patch").

`OracleNaivePatchUNet` restates distrifuser/models/naive_patch_sdxl.py on CPU in fp32: slice this rank's CFG half and
strip -> plain UNet -> gloo all_gather -> cat.  `run_naive_unet` drives it (impl="oracle") or the UNMODIFIED reference
NaivePatchUNet (impl="reference", through the diffusers stub; only where the reference tree exists) in the reference's
bring-up order, as harness.run_unet does for DistriUNetPP.  `run_naive_trajectory` is the denoising-loop counterpart of
harness.run_trajectory.  Running this module writes the naive-patch golden vectors from the reference:

    python -m oracle.naive_patch [--case NAME]
"""
from __future__ import annotations

import argparse
import dataclasses
import os
import tempfile
import time

import torch
from torch import distributed as dist
from torch import multiprocessing as mp

from oracle import harness


@dataclasses.dataclass(frozen=True)
class NaiveCase:
    """One naive-patch parity case (duck-types the fields of UNetCase that workloads.unet_inputs reads)."""
    name: str
    family: str = "tiny_sdxl"        # tiny_sdxl | tiny_sd15
    world_size: int = 2
    cfg: bool = True                 # do_classifier_free_guidance
    split_batch: bool = False
    scheme: str = "row"              # split_scheme: row | col | alternate
    steps: int = 4
    latent: int = 32                 # latent side S (image side = 8*S)
    weight_seed: int = 0
    input_seed: int = 1234

    @property
    def batch(self):
        return 2 if self.cfg else 1


NAIVE_CASES = (
    NaiveCase("naive_sdxl_w2_row", world_size=2, scheme="row"),                          # n=2, b=2
    NaiveCase("naive_sdxl_w4_col_split", world_size=4, split_batch=True, scheme="col"),  # n=2, b=1 (CFG halves)
    NaiveCase("naive_sdxl_w2_alternate", world_size=2, scheme="alternate"),              # n=2, rows / columns by step
    NaiveCase("naive_sdxl_w4_alternate", world_size=4, scheme="alternate"),              # n=4
    NaiveCase("naive_sd15_w4_col", family="tiny_sd15", world_size=4, scheme="col"),      # n=4, SD1.x topology
    NaiveCase("naive_sdxl_w8_split_col", world_size=8, split_batch=True, scheme="col"),  # n=4, b=1
)


def naive_config(case, rank: int):
    from oracle import workloads as W
    cfg = W.DuckConfig(case.world_size, rank, height=8 * case.latent, width=8 * case.latent,
                       do_classifier_free_guidance=case.cfg, split_batch=case.split_batch)
    cfg.parallelism, cfg.split_scheme = "naive_patch", case.scheme
    return cfg


class OracleNaivePatchUNet:
    """slice -> UNet -> all_gather -> cat, with the reference's counter protocol (the scheme `alternate` splits rows on even
    calls and columns on odd ones)."""

    def __init__(self, unet, cfg):
        self.unet, self.cfg, self.counter = unet, cfg, 0
        self.config = unet.config

    def set_counter(self, c: int = 0):
        self.counter = c

    def split_dim(self) -> int:
        return {"row": 2, "col": 3, "alternate": 2 if self.counter % 2 == 0 else 3}[self.cfg.split_scheme]

    def __call__(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None):
        cfg = self.cfg
        dim = self.split_dim()
        self.counter += 1
        if cfg.world_size == 1:
            return self.unet(sample, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs, return_dict=False)[0]
        split = cfg.do_classifier_free_guidance and cfg.split_batch
        if split:
            i = cfg.batch_idx()
            sample, encoder_hidden_states = sample[i:i + 1], encoder_hidden_states[i:i + 1]
            if torch.is_tensor(timestep) and timestep.ndim > 0:
                timestep = timestep[i:i + 1]
            if added_cond_kwargs is not None:
                added_cond_kwargs = {k: v[i:i + 1] for k, v in added_cond_kwargs.items()}
        n = cfg.n_device_per_batch
        strip = sample.chunk(n, dim)[cfg.split_idx()].contiguous()
        out = self.unet(strip, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs, return_dict=False)[0]
        parts = [torch.empty_like(out) for _ in range(cfg.world_size)]
        dist.all_gather(parts, out.contiguous())
        if split:
            return torch.cat([torch.cat(parts[:n], dim), torch.cat(parts[n:], dim)], 0)
        return torch.cat(parts, dim)


def _naive_worker(rank, case, impl, port, outdir):
    harness._paths(impl)
    from oracle import workloads as W
    harness._init(rank, case.world_size, port)
    cfg = naive_config(case, rank)
    if case.world_size > 1:
        harness._groups(cfg)
    ucfg = W.unet_config(case.family)
    unet = W.make_unet(case.family, case.weight_seed)
    first = W.unet_inputs(case, 0, ucfg)
    outs = []
    with torch.no_grad():
        if impl == "reference":
            from distrifuser.models.naive_patch_sdxl import NaivePatchUNet
            from distrifuser.utils import PatchParallelismCommManager
            model = NaivePatchUNet(unet, cfg)
            if cfg.n_device_per_batch > 1:                                   # pipelines.py:131-141 (nothing registers)
                model.set_comm_manager(PatchParallelismCommManager(cfg))
                model.set_counter(0)
                model(**first, return_dict=False, record=True)
            model.set_counter(0)
            model(**first, return_dict=False, record=True)                    # pipelines.py:144-145
            model.set_counter(0)                                              # pipelines.py:57
            for t in range(case.steps):
                outs.append(model(**W.unet_inputs(case, t, ucfg), return_dict=False)[0].clone())
        else:
            model = OracleNaivePatchUNet(unet, cfg)
            model.set_counter(0)
            for t in range(case.steps):
                outs.append(model(**W.unet_inputs(case, t, ucfg)).clone())
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_naive_unet(case, impl="oracle"):
    """-> outs[step] = eps prediction [B,4,S,S] (asserted identical on every rank)."""
    with tempfile.TemporaryDirectory() as d:
        if case.world_size == 1:
            _naive_worker(0, case, impl, 0, d)
        else:
            mp.spawn(_naive_worker, args=(case, impl, harness.free_port(), d), nprocs=case.world_size, join=True)
        per_rank = [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(case.world_size)]
    for r in range(1, case.world_size):
        for a, b in zip(per_rank[0], per_rank[r]):
            assert torch.equal(a, b), "final output must be identical on all ranks"
    return per_rank[0]


def _traj_worker(rank, case, port, outdir, num_steps, guidance):
    harness._paths("oracle")
    from oracle import workloads as W
    from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline
    harness._init(rank, case.world_size, port)
    cfg = naive_config(case, rank)
    if case.world_size > 1:
        harness._groups(cfg)
    ucfg = W.unet_config(case.family)
    model = OracleNaivePatchUNet(W.make_unet(case.family, case.weight_seed), cfg)
    pipe = SyntheticLatentPipeline(harness._OracleUNetAdapter(model, model.config),
                                   sdxl=ucfg.get("addition_embed_type") == "text_time", device="cpu", dtype=torch.float32)
    model.set_counter(0)
    g = torch.Generator().manual_seed(case.input_seed)
    with torch.no_grad():
        lat = pipe(prompt="a photo", height=8 * case.latent, width=8 * case.latent, num_inference_steps=num_steps,
                   guidance_scale=guidance, generator=g).images
    torch.save(lat, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_naive_trajectory(case, num_steps=8, guidance=5.0):
    """Final latents of a `num_steps` Euler trajectory with the naive-patch ORACLE UNet (fp32 CPU) -> [1,4,S,S]."""
    with tempfile.TemporaryDirectory() as d:
        if case.world_size == 1:
            _traj_worker(0, case, 0, d, num_steps, guidance)
        else:
            mp.spawn(_traj_worker, args=(case, harness.free_port(), d, num_steps, guidance), nprocs=case.world_size,
                     join=True)
        outs = [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(case.world_size)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    return outs[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    a = ap.parse_args()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    golden = os.path.join(root, "tests", "golden")
    os.makedirs(golden, exist_ok=True)
    for case in NAIVE_CASES:
        if a.case and case.name != a.case:
            continue
        t0 = time.time()
        outs = run_naive_unet(case, impl="reference")
        torch.save({"case": case.__dict__, "outs": [o.clone() for o in outs],
                    "source": "reference NaivePatchUNet @ /root/reference over oracle/diffusers_stub, gloo, fp32"},
                   os.path.join(golden, f"{case.name}.pt"))
        print(f"{case.name}: {time.time() - t0:.1f}s  std={outs[-1].std():.4f}", flush=True)


if __name__ == "__main__":
    main()
