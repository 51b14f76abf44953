"""TEST INFRASTRUCTURE (oracle) -- the naive patch baseline (parallelism="naive_patch").

`OracleNaivePatchUNet` restates distrifuser/models/naive_patch_sdxl.py on CPU in fp32: slice this rank's CFG half and
strip -> plain UNet -> gloo all_gather -> cat.  oracle/harness.py drives it (impl="oracle"), or the UNMODIFIED reference
NaivePatchUNet (impl="reference"), for a NaiveCase: `run_naive_unet` / `run_naive_trajectory` are harness.run_unet /
harness.run_trajectory under the names the naive-patch tests use.  `python -m oracle.make_golden --only naive` writes the
naive-patch golden vectors from the reference.
"""
from __future__ import annotations

import dataclasses

import torch
from torch import distributed as dist

from oracle.harness import run_trajectory as run_naive_trajectory  # noqa: F401
from oracle.harness import run_unet as run_naive_unet  # noqa: F401


@dataclasses.dataclass(frozen=True)
class NaiveCase:
    """One naive-patch parity case (the drivers read it through `batch`, `hw` and `config_kwargs()`, as for UNetCase)."""
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

    @property
    def hw(self):
        return self.latent, self.latent

    def config_kwargs(self) -> dict:
        return dict(height=8 * self.latent, width=8 * self.latent, do_classifier_free_guidance=self.cfg,
                    split_batch=self.split_batch, parallelism="naive_patch", split_scheme=self.scheme)


NAIVE_CASES = (
    NaiveCase("naive_sdxl_w2_row", world_size=2, scheme="row"),                          # n=2, b=2
    NaiveCase("naive_sdxl_w4_col_split", world_size=4, split_batch=True, scheme="col"),  # n=2, b=1 (CFG halves)
    NaiveCase("naive_sdxl_w2_alternate", world_size=2, scheme="alternate"),              # n=2, rows / columns by step
    NaiveCase("naive_sdxl_w4_alternate", world_size=4, scheme="alternate"),              # n=4
    NaiveCase("naive_sd15_w4_col", family="tiny_sd15", world_size=4, scheme="col"),      # n=4, SD1.x topology
    NaiveCase("naive_sdxl_w8_split_col", world_size=8, split_batch=True, scheme="col"),  # n=4, b=1
)


class OracleNaivePatchUNet:
    """slice -> UNet -> all_gather -> cat, with the reference's counter protocol (the scheme `alternate` splits rows on even
    calls and columns on odd ones)."""

    def __init__(self, unet, cfg):
        self.unet, self.cfg, self.counter = unet, cfg, 0
        self.config = unet.config

    def set_counter(self, c: int = 0):
        self.counter = c

    def prepare(self, inputs):
        """Nothing to size or pre-run: naive patch registers no buffers."""

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
