"""ControlNetModel for environments without `diffusers`: the module tree and state-dict keys of diffusers 0.24's
ControlNetModel for the SD1.x / SDXL configurations, built from the same blocks as the compat UNet, so that a real
checkpoint's state_dict loads with strict=True and DistriControlNetPP's surgery finds the layers it wraps.

A ControlNet is a copy of the UNet's encoder (conv_in, time / add embeddings, down blocks, mid block) plus a small conditioning
network on the pixel-resolution image and one zero-initialised 1x1 conv per UNet skip connection.  Its outputs line up pixel
for pixel with the UNet's skips; the UNet adds them (UNet2DConditionModel.forward, down_block_additional_residuals)."""
from __future__ import annotations

from types import SimpleNamespace

import torch
from torch import nn
from torch.nn import functional as F

from .unet_2d_condition import SDXL, TimestepEmbedding, UNet2DConditionModel, _Down, _Mid, embed

COND_CHANNELS = (16, 32, 96, 256)


def _zero(m: nn.Module) -> nn.Module:
    for p in m.parameters():
        nn.init.zeros_(p)
    return m


class ControlNetConditioningEmbedding(nn.Module):
    """3 -> 16 conv, then per width a 3x3 conv and a stride-2 3x3 conv (SiLU after each), then a zero conv to the UNet width:
    the conditioning image goes from pixel resolution to latent resolution (three stride-2 convs = the VAE's factor 8)."""

    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int = 3,
                 block_out_channels=COND_CHANNELS):
        super().__init__()
        self.conv_in = nn.Conv2d(conditioning_channels, block_out_channels[0], 3, padding=1)
        self.blocks = nn.ModuleList()
        for cin, cout in zip(block_out_channels[:-1], block_out_channels[1:]):
            self.blocks.append(nn.Conv2d(cin, cin, 3, padding=1))
            self.blocks.append(nn.Conv2d(cin, cout, 3, padding=1, stride=2))
        self.conv_out = _zero(nn.Conv2d(block_out_channels[-1], conditioning_embedding_channels, 3, padding=1))

    def forward(self, cond):
        x = F.silu(self.conv_in(cond))
        for blk in self.blocks:
            x = F.silu(blk(x))
        return self.conv_out(x)


class ControlNetModel(nn.Module):
    def __init__(self, conditioning_channels: int = 3, conditioning_embedding_out_channels=COND_CHANNELS, **overrides):
        super().__init__()
        cfg = dict(SDXL)
        cfg.update(overrides)
        self.config = SimpleNamespace(**cfg)
        c = self.config
        boc, g, eps = tuple(c.block_out_channels), c.norm_num_groups, c.norm_eps
        temb = boc[0] * 4
        heads, depth = tuple(c.attention_head_dim), tuple(c.transformer_layers_per_block)
        nb = len(boc)

        def attn_cfg(i, ch):
            return dict(heads=heads[i], head_dim=ch // heads[i], depth=depth[i], cross_dim=c.cross_attention_dim,
                        linear_proj=c.use_linear_projection)

        self.conv_in = nn.Conv2d(c.in_channels, boc[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        if c.addition_embed_type == "text_time":
            self.add_embedding = TimestepEmbedding(c.projection_class_embeddings_input_dim, temb)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(boc[0], conditioning_channels,
                                                                         tuple(conditioning_embedding_out_channels))
        self.down_blocks = nn.ModuleList()
        self.controlnet_down_blocks = nn.ModuleList([_zero(nn.Conv2d(boc[0], boc[0], 1))])
        ch = boc[0]
        for i, kind in enumerate(c.down_block_types):
            cin, ch = ch, boc[i]
            last = i == nb - 1
            self.down_blocks.append(_Down(cin, ch, temb, c.layers_per_block, g, eps, not last,
                                          attn_cfg(i, ch) if kind.startswith("CrossAttn") else None))
            for _ in range(c.layers_per_block + (0 if last else 1)):
                self.controlnet_down_blocks.append(_zero(nn.Conv2d(ch, ch, 1)))
        self.controlnet_mid_block = _zero(nn.Conv2d(boc[-1], boc[-1], 1))
        self.mid_block = _Mid(boc[-1], temb, g, eps, attn_cfg(nb - 1, boc[-1]))

    # time_emb_proj of every ResnetBlock2D as one GEMM per call, exactly as in the UNet
    _resnets = UNet2DConditionModel._resnets
    _batched_temb = UNet2DConditionModel._batched_temb

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @classmethod
    def from_unet(cls, unet: UNet2DConditionModel, conditioning_channels: int = 3,
                  conditioning_embedding_out_channels=COND_CHANNELS) -> "ControlNetModel":
        """A ControlNet whose encoder starts as a copy of `unet`'s (diffusers' ControlNetModel.from_unet): conv_in, the
        time / add embeddings, the down blocks and the mid block; the conditioning network and the zero convs are fresh."""
        cn = cls(conditioning_channels, conditioning_embedding_out_channels, **vars(unet.config))
        cn = cn.to(device=unet.conv_in.weight.device, dtype=unet.dtype)
        for name in ("conv_in", "time_embedding", "add_embedding", "down_blocks", "mid_block"):
            if hasattr(cn, name):
                getattr(cn, name).load_state_dict(getattr(unet, name).state_dict(), strict=True)
        return cn

    def zero_convs(self):
        return [*self.controlnet_down_blocks, self.controlnet_mid_block]

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                added_cond_kwargs=None, return_dict=False):
        """-> (down_block_res_samples, mid_block_res_sample), each multiplied by conditioning_scale (a float, or a device
        tensor of one element that a captured graph re-reads on every replay)."""
        emb = embed(self, sample, timestep, added_cond_kwargs)
        x = self.conv_in(sample) + self.controlnet_cond_embedding(controlnet_cond)
        skips = [x]
        for blk in self.down_blocks:
            x, s = blk(x, emb, encoder_hidden_states)
            skips += s
        x = self.mid_block(x, emb, encoder_hidden_states)
        if x.is_cuda and x.dtype == torch.float16:
            from .. import ops
            if not torch.is_tensor(conditioning_scale):
                conditioning_scale = torch.full((1,), float(conditioning_scale), dtype=torch.float32, device=x.device)
            outs = ops.controlnet_zero_convs(skips + [x], self.zero_convs(), conditioning_scale.float().reshape(1))
        else:
            outs = [conv(h) * conditioning_scale for conv, h in zip(self.zero_convs(), skips + [x])]
        return outs[:-1], outs[-1]
