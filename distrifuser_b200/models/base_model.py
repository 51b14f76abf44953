"""Reference: distrifuser/models/base_model.py:8-52 (same attributes and methods), plus the per-call protocol that
DistriUNetPP and NaivePatchUNet share (distri_sdxl_unet_pp.py:42-214 / naive_patch_sdxl.py:27-219).

The reference derives BaseModel from diffusers' (ModelMixin, ConfigMixin): StableDiffusion(XL)Pipeline.from_pretrained(...,
unet=DistriUNetPP) type-checks the component against ModelMixin.  When diffusers is importable the same bases are used
here; without it (this image) a plain nn.Module carries the `dtype` / `device` properties the mixin would provide."""
import torch
from torch import nn

from .. import _lib
from ..modules.base_module import BaseModule, nvtx_range
from ..utils import DistriConfig, PatchParallelismCommManager

try:  # pragma: no cover - depends on the environment
    from diffusers import ConfigMixin, ModelMixin
    _BASES = (ModelMixin, ConfigMixin)
except Exception:
    _BASES = (nn.Module,)


def _output_cls():
    try:
        from diffusers.models.unet_2d_condition import UNet2DConditionOutput
    except Exception:
        from ..compat.unet_2d_condition import UNet2DConditionOutput
    return UNet2DConditionOutput


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


def load_static_inputs(si: dict, sample, timestep, encoder_hidden_states, added_cond_kwargs, controlnet_cond=None) -> None:
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
    if controlnet_cond is not None and controlnet_cond is not si["controlnet_cond"]:
        si["controlnet_cond"].copy_(controlnet_cond)


class BaseModel(*_BASES):
    """A wrapper supplies what differs between the parallelisms: `_strip` (the UNet input of this rank and where its output
    lands in the image), `_step_kind`, `_graph_idx`, and the counters the pipeline pre-runs and captures."""

    def __init__(self, model: nn.Module, distri_config: DistriConfig):
        super(BaseModel, self).__init__()
        self.model = model
        self.distri_config = distri_config
        self.comm_manager = None
        self.buffer_list = None
        self.output_buffer = None
        self.counter = 0
        # for cuda graph
        self.static_inputs = None
        self.static_outputs = None
        self.cuda_graphs = None
        self.graph_launches = None       # number of this package's kernels inside each captured graph
        self.controlnet = None           # DistriControlNetPP run inside forward() (DistriUNetPP only)
        self._cn_scale = None            # device fp32 [1] set with the ControlNet: the scale the zero-conv kernel reads

    def _wrapped_modules(self):
        models = [self.model] if self.controlnet is None else [self.controlnet.model, self.model]
        return [m for model in models for m in model.modules() if isinstance(m, BaseModule)]

    def _controlnet_inputs(self, b, h, w, controlnet_cond, conditioning_scale):
        """Checks the conditioning image against the latent and loads the scale into the device scalar the graphs read."""
        if self.controlnet is None:
            if controlnet_cond is not None:
                raise ValueError("controlnet_cond was given but this UNet has no ControlNet attached (pass controlnet=... to "
                                 "from_synthetic or DistriUNetPP)")
            return None
        if controlnet_cond is None:
            raise ValueError("this UNet has a ControlNet attached: pass the conditioning image as controlnet_cond=[B, 3, H, W]")
        want = (b, self.controlnet.model.controlnet_cond_embedding.conv_in.module.in_channels, 8 * h, 8 * w)
        if tuple(controlnet_cond.shape) != want:
            raise ValueError(f"controlnet_cond has shape {tuple(controlnet_cond.shape)}; the {b}x4x{h}x{w} latent needs the "
                             f"conditioning image at pixel resolution, {want}")
        if conditioning_scale is not self._cn_scale:                 # a graph capture passes the device scalar itself
            if torch.is_tensor(conditioning_scale):
                self._cn_scale.copy_(conditioning_scale.reshape(1))
            else:
                self._cn_scale.fill_(float(conditioning_scale))
        return self._cn_scale

    def _strip(self, sample):
        """-> (UNet input of this rank, (row0, col0, hs, ws): the rows and columns of the image its output covers)."""
        raise NotImplementedError

    def _step_kind(self) -> int:
        """df_step_begin kind of the current counter: 0 = synchronous, 1 = asynchronous, 2 = frozen."""
        raise NotImplementedError

    def _graph_idx(self) -> int:
        """Captured graph that serves the current counter (an index into graph_counters())."""
        raise NotImplementedError

    def prerun_counters(self) -> list[int]:
        """Counters the pipeline runs eagerly before capturing, so that library autotuning and scratch allocations happen
        outside the capture."""
        raise NotImplementedError

    def graph_counters(self) -> list[int]:
        """Counters at which the pipeline captures one CUDA graph each."""
        raise NotImplementedError

    @nvtx_range()
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
        controlnet_cond=None,
        conditioning_scale=1.0,
        return_dict: bool = True,
        record: bool = False,
    ):
        """`controlnet_cond` ([B, 3, H, W] fp16) and `conditioning_scale` (a float or a device scalar) are not diffusers
        arguments: with a ControlNet attached, forward() runs it on this rank's strip and hands its residual strips to the UNet."""
        cfg = self.distri_config
        b, c, h, w = sample.shape
        if down_block_additional_residuals is not None or mid_block_additional_residual is not None:
            raise ValueError("residuals from outside cannot be used: each rank runs the UNet on its own strip, on one epoch per "
                             "denoising step, and a ControlNet called separately would advance that clock twice per step; attach "
                             "the ControlNet to the UNet (controlnet=...) and pass controlnet_cond=... instead")
        assert (class_labels is None and timestep_cond is None and attention_mask is None
                and cross_attention_kwargs is None and down_intrablock_additional_residuals is None
                and encoder_attention_mask is None)                  # distri_sdxl_unet_pp.py:63-72
        scale = self._controlnet_inputs(b, h, w, controlnet_cond, conditioning_scale)
        split = cfg.world_size > 1 and cfg.do_classifier_free_guidance and cfg.split_batch
        if split:
            assert b == 2
            sample, timestep, encoder_hidden_states, added_cond_kwargs = cfg_branch(
                cfg, sample, timestep, encoder_hidden_states, added_cond_kwargs)
            if controlnet_cond is not None:
                controlnet_cond = controlnet_cond[cfg.batch_idx():cfg.batch_idx() + 1]
        B = 2 if split else b

        if cfg.use_cuda_graph and not record and self.cuda_graphs is not None:
            load_static_inputs(self.static_inputs, sample, timestep, encoder_hidden_states, added_cond_kwargs, controlnet_cond)
            graph_idx = self._graph_idx()                            # distri_sdxl_unet_pp.py:108-113
            self.cuda_graphs[graph_idx].replay()
            if self.graph_launches is not None:
                _lib.LAUNCHES["total"] += self.graph_launches[graph_idx]
            output = self.static_outputs[graph_idx]
        else:
            cm = self.comm_manager
            live = cm is not None and cm.arena is not None
            if cm is not None and cm.arena is None and cfg.world_size > 1 and cm.output_spec is None:
                cm.register_output(B, c, h, w)
            if live:
                cm.step_begin(self._step_kind())
            # NHWC inside the UNet; `sample` itself stays the (sliced) view of the caller's tensor so that a captured
            # graph re-reads the static input on every replay
            x, (row0, col0, hs, ws) = self._strip(sample)
            x = x.contiguous(memory_format=torch.channels_last)
            residuals = {}
            if self.controlnet is not None:                          # ControlNet first: it registers and publishes first
                down, mid = self.controlnet(x, timestep, encoder_hidden_states,
                                            controlnet_cond.contiguous(memory_format=torch.channels_last), scale,
                                            added_cond_kwargs=added_cond_kwargs)
                residuals = dict(down_block_additional_residuals=down, mid_block_additional_residual=mid)
            output = self.model(x, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs, return_dict=False,
                                **residuals)[0]
            if cfg.world_size > 1 and live:                          # distri_sdxl_unet_pp.py:162-169 / 186-193
                # Every rank waits here for the strips of every world rank: the gather is a per-call world barrier, which
                # is what keeps the output banks safe to reuse (BANK-REUSE INVARIANT in utils.py).
                if self.output_buffer is None:
                    self.output_buffer = torch.empty((B, c, h, w), device=output.device, dtype=output.dtype)
                strip = output.contiguous()
                bs = strip.shape[0]
                assert tuple(strip.shape) == (bs, c, hs, ws)
                batch0 = cfg.batch_idx() if split else 0
                _lib.check(_lib.lib().df_output_gather_2d(cm.world, strip.data_ptr(), self.output_buffer.data_ptr(),
                                                          B, c, h, w, bs, hs, ws, batch0, row0, col0, 0, cm.output_off,
                                                          torch.cuda.current_stream().cuda_stream), "df_output_gather_2d")
                output = self.output_buffer
            elif cfg.world_size > 1:
                # registration pass: buffers do not exist yet, the value is never consumed
                output = output.new_zeros((B, c, h, w))
            if cm is not None:
                cm.join()
            if record:
                if self.static_inputs is None:                       # distri_sdxl_unet_pp.py:194-201
                    self.static_inputs = {"sample": sample, "timestep": timestep,
                                          "encoder_hidden_states": encoder_hidden_states,
                                          "added_cond_kwargs": added_cond_kwargs, "controlnet_cond": controlnet_cond,
                                          "conditioning_scale": scale}
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

    def set_counter(self, counter: int = 0):                        # base_model.py:27-31
        self.counter = counter
        for module in self._wrapped_modules():
            module.set_counter(counter)

    def set_comm_manager(self, comm_manager: PatchParallelismCommManager):   # base_model.py:33-37
        self.comm_manager = comm_manager
        for module in self._wrapped_modules():
            module.set_comm_manager(comm_manager)

    def setup_cuda_graph(self, static_outputs, cuda_graphs, graph_launches=None):   # base_model.py:39-41
        self.static_outputs = static_outputs
        self.cuda_graphs = cuda_graphs
        self.graph_launches = graph_launches

    @property
    def config(self):
        return self.model.config

    def synchronize(self):                                         # base_model.py:47-52
        if self.comm_manager is not None:
            self.comm_manager.join()


def _first_param(m: nn.Module):
    for p in m.parameters():
        return p
    for b in m.buffers():
        return b
    return None


if not any(hasattr(b, "dtype") for b in _BASES):                   # ModelMixin.dtype / .device for the nn.Module fallback
    BaseModel.dtype = property(lambda self: getattr(_first_param(self), "dtype", torch.float32))
    BaseModel.device = property(lambda self: getattr(_first_param(self), "device", torch.device("cpu")))
