"""DistriUNetPP -- drop-in for distrifuser/models/distri_sdxl_unet_pp.py:15-214 (patch-parallel UNet wrapper).

Same constructor, forward signature (including the non-diffusers `record` kwarg), counter protocol, CFG batch
split and three-graph replay as the reference.  Differences, all internal:
  * the wrappers are installed for every world size (the reference leaves world_size==1 unwrapped, :18), so the
    sm_90a kernels are the only attention / GroupNorm path;
  * the final epsilon all_gather + cat (:162-169,186-193) is df_output_gather_2d (BaseModel.forward): each rank stores
    its strip into every peer's arena and waits on flags;
  * GroupNorm -> SiLU pairs of ResnetBlock2D / conv_norm_out run fused inside the GroupNorm kernel.
"""
import torch
from torch import nn

from ..modules.base_module import BaseModule
from ..modules.pp.attn import DistriCrossAttentionPP, DistriSelfAttentionPP
from ..modules.pp.conv2d import DistriConv2dPP
from ..modules.pp.groupnorm import DistriGroupNorm
from ..utils import DistriConfig, patch_rows, row_offset, split_units
from .base_model import BaseModel


def _is_attention(m: nn.Module) -> bool:
    return all(hasattr(m, a) for a in ("to_q", "to_k", "to_v", "to_out", "heads"))


def install_pp_wrappers(model: nn.Module, distri_config) -> None:
    """Module surgery of distri_sdxl_unet_pp.py:19-40 in place: 3x3 convs, self / cross attention and GroupNorm become the
    sm_90a wrappers, GroupNorm -> SiLU pairs fuse, and the UNet goes channels_last.  The wrappers read the patch layout from
    `distri_config` (NaivePatchUNet passes a one-patch view of its config)."""
    for name, module in list(model.named_modules()):
        if isinstance(module, BaseModule):
            continue
        for subname, submodule in list(module.named_children()):
            if isinstance(submodule, nn.Conv2d):
                k = submodule.kernel_size
                if k == (1, 1) or k == 1:
                    continue
                setattr(module, subname, DistriConv2dPP(submodule, distri_config, is_first_layer=subname == "conv_in"))
            elif _is_attention(submodule):
                if subname == "attn1":
                    setattr(module, subname, DistriSelfAttentionPP(submodule, distri_config))
                else:
                    assert subname == "attn2"
                    setattr(module, subname, DistriCrossAttentionPP(submodule, distri_config))
            elif isinstance(submodule, nn.GroupNorm):
                setattr(module, subname, DistriGroupNorm(submodule, distri_config))
    # GroupNorm -> SiLU fusion where the block exposes the switch (compat UNet; diffusers blocks keep SiLU separate)
    for module in model.modules():
        if hasattr(module, "fused_norm_act"):
            module.fused_norm_act = True
            for nm in ("norm1", "norm2", "conv_norm_out"):
                sub = getattr(module, nm, None)
                if isinstance(sub, DistriGroupNorm):
                    sub.fuse_silu = True
    model.to(memory_format=torch.channels_last)


def downsample_factor(model: nn.Module) -> int:
    """u = 2^(stride-2 downsamplers of the UNet): latent rows per row unit, so that every level holds whole rows of each unit."""
    blocks = getattr(model, "down_blocks", None)
    if blocks is None:
        return 2 ** (len(model.config.block_out_channels) - 1)
    return 2 ** sum(1 for blk in blocks if getattr(blk, "downsamplers", None) is not None)


def row_plan(model: nn.Module, cfg: DistriConfig) -> list[int]:
    """Units of latent rows of each patch rank (utils.split_units): rank r of n holds U // n or U // n + 1 consecutive units
    of u rows, U = latent rows / u.  Raises ValueError for a height that cannot be split."""
    n = cfg.n_device_per_batch
    rows, u = cfg.height // 8, downsample_factor(model)
    if rows % u != 0:
        raise ValueError(f"patch parallelism needs the latent height to be a multiple of {u} (2^downsamplers of the UNet): "
                         f"height {cfg.height} gives {rows} latent rows")
    if rows // u < n:
        raise ValueError(f"patch parallelism over {n} ranks needs at least {n} units of {u} latent rows: height {cfg.height} "
                         f"gives {rows // u}")
    return split_units(rows // u, n)


class DistriUNetPP(BaseModel):  # for Patch Parallelism
    def __init__(self, model: nn.Module, distri_config: DistriConfig, controlnet: nn.Module | None = None):
        """`controlnet` (optional): a ControlNetModel (or DistriControlNetPP) that forward() runs on this rank's strip before the
        UNet, on the same epoch; its residuals go into the UNet without leaving the rank."""
        # the row plan (uneven strips when n does not divide the row units); one patch keeps the whole image, any height
        row_units = row_plan(model, distri_config) if distri_config.n_device_per_batch > 1 else None
        install_pp_wrappers(model, distri_config)
        super().__init__(model, distri_config)
        self.row_units = row_units
        for module in model.modules():
            if isinstance(module, BaseModule):
                module.row_units = self.row_units
        if controlnet is not None:
            from .distri_controlnet_pp import DistriControlNetPP
            if not isinstance(controlnet, DistriControlNetPP):
                controlnet = DistriControlNetPP(controlnet, distri_config)
            assert controlnet.row_units == self.row_units, (controlnet.row_units, self.row_units)
            self.controlnet = controlnet
            self._cn_scale = torch.ones(1, dtype=torch.float32, device=distri_config.device)

    def _strip(self, sample):
        h, w = sample.shape[2:]
        if self.row_units is None:                                   # one patch: the whole image
            return sample, (0, 0, h, w)
        units, r = self.row_units, self.distri_config.split_idx()
        hs = h * units[r] // sum(units)
        # the whole latent goes in (conv_in takes this rank's rows); the output is this rank's strip of full-width rows
        return sample, (row_offset(patch_rows(units, r, hs), r), 0, hs, w)

    def _step_kind(self) -> int:
        cfg = self.distri_config
        if self.counter <= cfg.warmup_steps or cfg.mode == "full_sync":
            return 0
        return 2 if cfg.mode == "no_sync" else 1

    def _graph_idx(self) -> int:
        w = self.distri_config.warmup_steps
        return 0 if self.counter <= w else (1 if self.counter == w + 1 else 2)

    def prerun_counters(self) -> list[int]:
        return [0]

    def graph_counters(self) -> list[int]:
        """Synchronous step, first asynchronous step, steady state (pipelines.py:147-165)."""
        w = self.distri_config.warmup_steps
        return [0, w + 1, w + 2]
