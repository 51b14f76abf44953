"""NaivePatchUNet -- drop-in for distrifuser/models/naive_patch_sdxl.py:10-219 (the naive patch baseline).

Every rank runs the plain UNet on its own strip of the latent (rows, columns, or rows and columns on alternate steps) and
talks to no peer until the final epsilon gather.  Same constructor, forward signature (including `record`), counter protocol,
CFG batch split and graph choice as the reference.  A naive-patch rank is a one-patch DistriUNetPP rank that runs on a
strip: the same sm_90a wrappers are installed, but they see a one-patch view of the config and no comm manager, so they
take their local paths (GroupNorm statistics of the strip, attention over the strip's tokens, zero-padded convs).  The
all_gather + cat of the reference (:151-154,195-197) is df_output_gather_2d."""
import copy

import torch
from torch import nn

from .. import _lib
from ..modules.base_module import nvtx_range
from ..utils import DistriConfig, PatchParallelismCommManager
from .base_model import BaseModel
from .distri_sdxl_unet_pp import _output_cls, cfg_branch, install_pp_wrappers, load_static_inputs


class NaivePatchUNet(BaseModel):  # for Patch Parallelism
    def __init__(self, model: nn.Module, distri_config: DistriConfig):
        one_patch = copy.copy(distri_config)
        one_patch.n_device_per_batch = 1                             # split_idx() == 0: the wrappers' local paths
        install_pp_wrappers(model, one_patch)
        super().__init__(model, distri_config)

    def set_comm_manager(self, comm_manager: PatchParallelismCommManager):
        # the only communication is the output gather, done here: the modules keep comm_manager None
        self.comm_manager = comm_manager

    def _split_dim(self) -> int:
        scheme = self.distri_config.split_scheme                     # naive_patch_sdxl.py:115-122 / 157-164
        if scheme == "row":
            return 2
        if scheme == "col":
            return 3
        if scheme == "alternate":
            return 2 if self.counter % 2 == 0 else 3
        raise NotImplementedError(scheme)

    @nvtx_range("NaivePatchUNet")
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
                and encoder_attention_mask is None)                  # naive_patch_sdxl.py:34-43
        split = cfg.world_size > 1 and cfg.do_classifier_free_guidance and cfg.split_batch
        if split:                                                    # naive_patch_sdxl.py:47-58 / 101-113
            assert b == 2
            sample, timestep, encoder_hidden_states, added_cond_kwargs = cfg_branch(
                cfg, sample, timestep, encoder_hidden_states, added_cond_kwargs)

        if cfg.use_cuda_graph and not record and self.cuda_graphs is not None:
            load_static_inputs(self.static_inputs, sample, timestep, encoder_hidden_states, added_cond_kwargs)
            graph_idx = self.counter % 2 if cfg.split_scheme == "alternate" else 0   # naive_patch_sdxl.py:79-81
            self.cuda_graphs[graph_idx].replay()
            if self.graph_launches is not None:
                _lib.LAUNCHES["total"] += self.graph_launches[graph_idx]
            output = self.static_outputs[graph_idx]
        else:
            n, r = cfg.n_device_per_batch, cfg.split_idx()
            dim = self._split_dim()
            bs = sample.shape[0]
            hs, ws = (h // n, w) if dim == 2 else (h, w // n)
            row0, col0 = (r * hs, 0) if dim == 2 else (0, r * ws)
            # NHWC inside the UNet; `sample` itself stays the (sliced) view of the caller's tensor so that a captured graph
            # re-reads the static input on every replay
            strip = sample[:, :, row0:row0 + hs, col0:col0 + ws].contiguous(memory_format=torch.channels_last)
            cm = self.comm_manager
            live = cm is not None and cm.arena is not None
            B = 2 if split else b
            if cm is not None and cm.arena is None and cfg.world_size > 1 and cm.output_spec is None:
                cm.register_output(B, c, h, w)                       # the arena holds the output image only
            if live:
                cm.step_begin(2)                                     # frozen: only the output epoch clock[2] advances
            output = self.model(strip, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs,
                                return_dict=False)[0]
            if cfg.world_size > 1 and live:
                # Every rank waits here for the strips of every world rank: the gather is a per-call world barrier, which
                # is what keeps the output banks safe to reuse (BANK-REUSE INVARIANT in utils.py).
                if self.output_buffer is None:
                    self.output_buffer = torch.empty((B, c, h, w), device=output.device, dtype=output.dtype)
                out_strip = output.contiguous()
                assert tuple(out_strip.shape) == (bs, c, hs, ws)
                batch0 = cfg.batch_idx() if split else 0
                _lib.check(_lib.lib().df_output_gather_2d(cm.world, out_strip.data_ptr(), self.output_buffer.data_ptr(),
                                                          B, c, h, w, bs, hs, ws, batch0, row0, col0, 0, cm.output_off,
                                                          torch.cuda.current_stream().cuda_stream), "df_output_gather_2d")
                output = self.output_buffer
            elif cfg.world_size > 1:
                # registration pass: buffers do not exist yet, the value is never consumed
                output = output.new_zeros((B, c, h, w))
            if cm is not None:
                cm.join()
            if record:
                if self.static_inputs is None:                       # naive_patch_sdxl.py:199-206
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
