"""DistriControlNetPP -- a ControlNet made patch-parallel with the same sm_90a wrappers as the UNet.

Its 3x3 convs (the conditioning network's included), self / cross attention and GroupNorm become DistriConv2dPP /
DistriSelfAttentionPP / DistriCrossAttentionPP / DistriGroupNorm, with one-step-stale halos, K/V and statistics like the UNet's.
The 1x1 zero convs stay strip-local (install_pp_wrappers skips 1x1 convs) and run as one kernel per call
(ops.controlnet_zero_convs).  The residuals line up pixel for pixel with the UNet's skips, so rank r's residual strips are
exactly the rows its UNet strip needs: they never leave the rank.

The ControlNet is not called on its own: DistriUNetPP runs it inside its forward, after df_step_begin, so that both models
share one epoch per denoising step and the end-of-call output gather (the bank-reuse invariant in utils.py) covers both."""
from torch import nn

from ..modules.base_module import BaseModule
from ..utils import DistriConfig
from .distri_sdxl_unet_pp import install_pp_wrappers, row_plan


class DistriControlNetPP(nn.Module):
    def __init__(self, controlnet: nn.Module, distri_config: DistriConfig):
        super().__init__()
        # the UNet's row plan: a ControlNet has the UNet's encoder, so the same downsamplers; at pixel resolution a rank's strip
        # is 8x its latent rows, which the first-layer slice and patch_rows derive from the same units
        self.row_units = row_plan(controlnet, distri_config) if distri_config.n_device_per_batch > 1 else None
        install_pp_wrappers(controlnet, distri_config)
        self.model = controlnet
        self.distri_config = distri_config
        for module in self.wrappers():
            module.row_units = self.row_units

    def wrappers(self):
        return [m for m in self.model.modules() if isinstance(m, BaseModule)]

    @property
    def config(self):
        return self.model.config

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale, added_cond_kwargs=None):
        """sample: the whole latent, controlnet_cond: the whole [b, 3, 8h, 8w] image (each first conv takes this rank's rows)
        -> this rank's residual strips (down_block_res_samples, mid_block_res_sample)."""
        return self.model(sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale,
                          added_cond_kwargs=added_cond_kwargs)
