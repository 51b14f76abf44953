"""TEST INFRASTRUCTURE (oracle) -- not product code.

diffusers 0.24's ControlNetModel for the SD1.x / SDXL configurations, restated on this stub's UNet blocks with diffusers'
parameter names, so that the product's compat ControlNetModel loads its state_dict strict=True.  A ControlNet is a copy of
the UNet's encoder plus a conditioning network on the pixel-resolution image and one zero-initialised 1x1 conv per UNet skip;
the UNet adds its outputs (UNet2DConditionModel.forward, down_block_additional_residuals / mid_block_additional_residual).
"""
from __future__ import annotations

from types import SimpleNamespace

from torch import nn
from torch.nn import functional as F

from .unet_2d_condition import (CrossAttnDownBlock2D, DownBlock2D, TimestepEmbedding, Timesteps, UNetMidBlock2DCrossAttn,
                                embed, sdxl_config)


class ControlNetConditioningEmbedding(nn.Module):
    def __init__(self, emb_channels, cond_channels=3, block_out_channels=(16, 32, 96, 256)):
        super().__init__()
        self.conv_in = nn.Conv2d(cond_channels, block_out_channels[0], kernel_size=3, padding=1)
        self.blocks = nn.ModuleList([])
        for i in range(len(block_out_channels) - 1):
            cin, cout = block_out_channels[i], block_out_channels[i + 1]
            self.blocks.append(nn.Conv2d(cin, cin, kernel_size=3, padding=1))
            self.blocks.append(nn.Conv2d(cin, cout, kernel_size=3, padding=1, stride=2))
        self.conv_out = nn.Conv2d(block_out_channels[-1], emb_channels, kernel_size=3, padding=1)
        nn.init.zeros_(self.conv_out.weight)
        nn.init.zeros_(self.conv_out.bias)

    def forward(self, conditioning):
        embedding = F.silu(self.conv_in(conditioning))
        for block in self.blocks:
            embedding = F.silu(block(embedding))
        return self.conv_out(embedding)


def _zero_conv(c):
    conv = nn.Conv2d(c, c, kernel_size=1)
    nn.init.zeros_(conv.weight)
    nn.init.zeros_(conv.bias)
    return conv


class ControlNetModel(nn.Module):
    """diffusers 0.24 ControlNetModel for the SD1.x / SDXL configurations, without the options they leave off."""

    def __init__(self, **cfg):
        super().__init__()
        full = sdxl_config()
        full.update(cfg)
        self.config = SimpleNamespace(**full)
        c = self.config
        boc = tuple(c.block_out_channels)
        temb = boc[0] * 4
        g, eps = c.norm_num_groups, c.norm_eps
        heads, depth = tuple(c.attention_head_dim), tuple(c.transformer_layers_per_block)
        self.conv_in = nn.Conv2d(c.in_channels, boc[0], 3, padding=1)
        self.time_proj = Timesteps(boc[0], True, 0)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        if c.addition_embed_type == "text_time":
            self.add_time_proj = Timesteps(c.addition_time_embed_dim, True, 0)
            self.add_embedding = TimestepEmbedding(c.projection_class_embeddings_input_dim, temb)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(boc[0])
        self.down_blocks = nn.ModuleList([])
        self.controlnet_down_blocks = nn.ModuleList([_zero_conv(boc[0])])
        out_ch = boc[0]
        for i, t in enumerate(c.down_block_types):
            in_ch, out_ch = out_ch, boc[i]
            final = i == len(boc) - 1
            cls = CrossAttnDownBlock2D if t == "CrossAttnDownBlock2D" else DownBlock2D
            self.down_blocks.append(cls(in_ch, out_ch, temb, c.layers_per_block, g, eps, not final, heads=heads[i],
                                        depth=depth[i], cross_dim=c.cross_attention_dim, linear_proj=c.use_linear_projection))
            for _ in range(c.layers_per_block):
                self.controlnet_down_blocks.append(_zero_conv(out_ch))
            if not final:
                self.controlnet_down_blocks.append(_zero_conv(out_ch))
        self.controlnet_mid_block = _zero_conv(boc[-1])
        self.mid_block = UNetMidBlock2DCrossAttn(boc[-1], temb, g, eps, heads[-1], depth[-1], c.cross_attention_dim,
                                                 c.use_linear_projection)

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                added_cond_kwargs=None):
        """-> (down_block_res_samples, mid_block_res_sample), each multiplied by conditioning_scale."""
        emb = embed(self, sample, timestep, added_cond_kwargs)
        sample = self.conv_in(sample)
        sample = sample + self.controlnet_cond_embedding(controlnet_cond)
        down = (sample,)
        for blk in self.down_blocks:
            sample, res = blk(sample, emb, encoder_hidden_states=encoder_hidden_states)
            down += res
        sample = self.mid_block(sample, emb, encoder_hidden_states=encoder_hidden_states)
        down = [blk(s) * conditioning_scale for s, blk in zip(down, self.controlnet_down_blocks)]
        return down, self.controlnet_mid_block(sample) * conditioning_scale
