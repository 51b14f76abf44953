"""Reference: distrifuser/modules/base_module.py:6-29 (same attributes and state protocol)."""
import functools
import os

import torch
from torch import nn

from ..utils import DistriConfig, patch_rows

NVTX = os.environ.get("DF_NVTX", "1") != "0"     # NVTX range per wrapper call (SURVEY 5 tracing row); DF_NVTX=0 removes them


_HAS_CUDA = None


def nvtx_range(name: str | None = None):
    """Decorator: brackets a wrapper's forward with an NVTX range `name[idx]` (default name: the class of `self`) when CUDA is
    in use (shows up in nsys / ncu --nvtx; a no-op on captured-graph replays, where Python does not run)."""
    def deco(fn):
        if not NVTX:
            return fn

        @functools.wraps(fn)
        def wrapped(self, *args, **kwargs):
            global _HAS_CUDA
            if _HAS_CUDA is None:
                _HAS_CUDA = torch.cuda.is_available()
            if not _HAS_CUDA:
                return fn(self, *args, **kwargs)
            label, idx = name or type(self).__name__, getattr(self, "idx", None)
            torch.cuda.nvtx.range_push(label if idx is None else f"{label}[{idx}]")
            try:
                return fn(self, *args, **kwargs)
            finally:
                torch.cuda.nvtx.range_pop()
        return wrapped
    return deco


class BaseModule(nn.Module):
    def __init__(self, module: nn.Module, distri_config: DistriConfig):
        super().__init__()
        self.module = module
        self.distri_config = distri_config
        self.comm_manager = None
        self.counter = 0
        self.buffer_list = None
        self.idx = None
        self.row_units = None            # units of latent rows per patch rank (DistriUNetPP's row plan); None: equal strips
        self.allow_fp32 = False          # True: fp32 tensors are accepted too (the VAE decoder's upcast part)

    def forward(self, *args, **kwargs):
        raise NotImplementedError

    def patch_rows(self, h: int) -> list[int]:
        """Rows (or tokens) of every patch rank at the level where this rank holds h of them."""
        n = self.distri_config.n_device_per_batch
        return patch_rows(self.row_units or [1] * n, self.distri_config.split_idx(), h)

    def set_counter(self, counter: int = 0):
        self.counter = counter

    def set_comm_manager(self, comm_manager):
        self.comm_manager = comm_manager

    # -- helpers shared by the native wrappers
    def _is_sync_step(self) -> bool:
        """counter <= warmup_steps  (attn.py:132, conv2d.py:92, groupnorm.py:45)."""
        return self.counter <= self.distri_config.warmup_steps

    def _bound(self) -> bool:
        cm = self.comm_manager
        return cm is not None and cm.arena is not None and self.idx is not None

    def _recording(self) -> bool:
        cm = self.comm_manager
        return cm is not None and cm.arena is None

    def _require_cuda_half(self, x: torch.Tensor, who: str):
        if x.is_cuda and (x.dtype == torch.float16 or (self.allow_fp32 and x.dtype == torch.float32)):
            return
        what = "fp16 or fp32" if self.allow_fp32 else "fp16"
        raise RuntimeError(
            f"{who}: distrifuser_b200 runs {what} tensors on a CUDA device only (got {x.dtype} on {x.device}); "
            "there is no CPU / eager fallback")
