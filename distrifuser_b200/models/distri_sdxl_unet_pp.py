"""DistriUNetPP -- drop-in for distrifuser/models/distri_sdxl_unet_pp.py:15-214 (patch-parallel UNet wrapper).

Same constructor, forward signature (including the non-diffusers `record` kwarg), counter protocol, CFG batch
split and three-graph replay as the reference.  Differences, all internal:
  * the wrappers are installed for every world size (the reference leaves world_size==1 unwrapped, :18), so the
    sm_90a kernels are the only attention / GroupNorm path;
  * the final epsilon all_gather + cat (:162-169,186-193) is df_output_gather: each rank stores its strip into
    every peer's arena and waits on flags;
  * GroupNorm -> SiLU pairs of ResnetBlock2D / conv_norm_out run fused inside the GroupNorm kernel.
"""
import torch
from torch import nn

from .. import _lib
from ..modules.base_module import BaseModule, nvtx_range
from ..modules.pp.attn import DistriCrossAttentionPP, DistriSelfAttentionPP
from ..modules.pp.conv2d import DistriConv2dPP
from ..modules.pp.groupnorm import DistriGroupNorm
from ..utils import DistriConfig, patch_rows, row_offset, split_units
from .base_model import BaseModel


def _is_attention(m: nn.Module) -> bool:
    return all(hasattr(m, a) for a in ("to_q", "to_k", "to_v", "to_out", "heads"))


def _output_cls():
    try:
        from diffusers.models.unet_2d_condition import UNet2DConditionOutput
    except Exception:
        from ..compat.unet_2d_condition import UNet2DConditionOutput
    return UNet2DConditionOutput


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


def cfg_branch(cfg: DistriConfig, sample, timestep, encoder_hidden_states, added_cond_kwargs):
    """This rank's half of the CFG batch (distri_sdxl_unet_pp.py:77-87 / 134-146)."""
    i = cfg.batch_idx()
    sample = sample[i:i + 1]
    if torch.is_tensor(timestep) and timestep.ndim > 0:
        timestep = timestep[i:i + 1]
    encoder_hidden_states = encoder_hidden_states[i:i + 1]
    if added_cond_kwargs is not None:                                # new dict: the caller's is not mutated (SURVEY D-10)
        added_cond_kwargs = {k: v[i:i + 1] for k, v in added_cond_kwargs.items()}
    return sample, timestep, encoder_hidden_states, added_cond_kwargs


def load_static_inputs(si: dict, sample, timestep, encoder_hidden_states, added_cond_kwargs) -> None:
    """Copies a call's inputs into the captured graphs' static inputs (distri_sdxl_unet_pp.py:89-106)."""
    assert si["sample"].shape == sample.shape
    si["sample"].copy_(sample)
    if torch.is_tensor(timestep):
        si["timestep"].copy_(timestep.expand(si["timestep"].shape) if timestep.ndim == 0 else timestep)
    else:
        si["timestep"].fill_(timestep)                               # no .item() host sync (SURVEY A6)
    si["encoder_hidden_states"].copy_(encoder_hidden_states)
    if added_cond_kwargs is not None:
        for k in added_cond_kwargs:
            si["added_cond_kwargs"][k].copy_(added_cond_kwargs[k])


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
    def __init__(self, model: nn.Module, distri_config: DistriConfig):
        # the row plan (uneven strips when n does not divide the row units); one patch keeps the whole image, any height
        row_units = row_plan(model, distri_config) if distri_config.n_device_per_batch > 1 else None
        install_pp_wrappers(model, distri_config)
        super().__init__(model, distri_config)
        self.row_units = row_units
        for module in model.modules():
            if isinstance(module, BaseModule):
                module.row_units = self.row_units

    def _step_kind(self) -> int:
        cfg = self.distri_config
        if self.counter <= cfg.warmup_steps or cfg.mode == "full_sync":
            return 0
        return 2 if cfg.mode == "no_sync" else 1

    @nvtx_range("DistriUNetPP")
    def forward(
        self,
        sample: torch.FloatTensor,
        timestep,
        encoder_hidden_states: torch.Tensor,
        class_labels=None,
        timestep_cond=None,
        attention_mask=None,
        cross_attention_kwargs=None,
        added_cond_kwargs=None,
        down_block_additional_residuals=None,
        mid_block_additional_residual=None,
        down_intrablock_additional_residuals=None,
        encoder_attention_mask=None,
        return_dict: bool = True,
        record: bool = False,
    ):
        cfg = self.distri_config
        b, c, h, w = sample.shape
        assert (class_labels is None and timestep_cond is None and attention_mask is None
                and cross_attention_kwargs is None and down_block_additional_residuals is None
                and mid_block_additional_residual is None and down_intrablock_additional_residuals is None
                and encoder_attention_mask is None)                  # distri_sdxl_unet_pp.py:63-72
        split = cfg.world_size > 1 and cfg.do_classifier_free_guidance and cfg.split_batch
        if split:
            assert b == 2
            sample, timestep, encoder_hidden_states, added_cond_kwargs = cfg_branch(
                cfg, sample, timestep, encoder_hidden_states, added_cond_kwargs)

        if cfg.use_cuda_graph and not record and self.cuda_graphs is not None:
            load_static_inputs(self.static_inputs, sample, timestep, encoder_hidden_states, added_cond_kwargs)
            if self.counter <= cfg.warmup_steps:                     # distri_sdxl_unet_pp.py:108-113
                graph_idx = 0
            elif self.counter == cfg.warmup_steps + 1:
                graph_idx = 1
            else:
                graph_idx = 2
            self.cuda_graphs[graph_idx].replay()
            if self.graph_launches is not None:
                _lib.LAUNCHES["total"] += self.graph_launches[graph_idx]
            output = self.static_outputs[graph_idx]
        else:
            cm = self.comm_manager
            live = cm is not None and cm.arena is not None
            if cm is not None and cm.arena is None and cfg.world_size > 1 and cm.output_spec is None:
                cm.register_output(b if not split else 2, c, h, w)
            if live:
                cm.step_begin(self._step_kind())
            # NHWC inside the UNet; `sample` itself stays the (sliced) view of the caller's tensor so that a captured
            # graph re-reads the static input on every replay
            sample_cl = sample.contiguous(memory_format=torch.channels_last)
            output = self.model(sample_cl, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs,
                                return_dict=False)[0]
            if cfg.world_size > 1 and live:                          # distri_sdxl_unet_pp.py:162-169 / 186-193
                B = 2 if split else b
                n = cfg.n_device_per_batch
                if self.output_buffer is None:
                    self.output_buffer = torch.empty((B, c, h, w), device=output.device, dtype=output.dtype)
                strip = output.contiguous()
                bs, _, hs, _ = strip.shape
                batch0 = cfg.batch_idx() if split else 0
                row0 = row_offset(patch_rows(self.row_units, cfg.split_idx(), hs), cfg.split_idx()) if n > 1 else 0
                if n == 1:
                    assert hs == h
                _lib.check(_lib.lib().df_output_gather(cm.world, strip.data_ptr(), self.output_buffer.data_ptr(), B, c, h, w,
                                                       bs, hs, batch0, row0, 0, cm.output_off,
                                                       torch.cuda.current_stream().cuda_stream), "df_output_gather")
                output = self.output_buffer
            elif cfg.world_size > 1:
                # registration pass: buffers do not exist yet, the value is never consumed
                B = 2 if split else b
                output = output.new_zeros((B, c, h, w))
            if cm is not None:
                cm.join()
            if record:
                if self.static_inputs is None:                       # distri_sdxl_unet_pp.py:194-201
                    self.static_inputs = {"sample": sample, "timestep": timestep,
                                          "encoder_hidden_states": encoder_hidden_states,
                                          "added_cond_kwargs": added_cond_kwargs}
                self.synchronize()

        if return_dict:
            output = _output_cls()(sample=output)
        else:
            output = (output,)
        self.counter += 1
        return output

    @property
    def add_embedding(self):
        return self.model.add_embedding
