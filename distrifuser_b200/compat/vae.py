"""AutoencoderKL: the decoder half of diffusers 0.24's VAE (diffusers/models/autoencoder_kl.py, vae.py Decoder,
unet_2d_blocks.py UNetMidBlock2D / UpDecoderBlock2D, resnet.py ResnetBlock2D / Upsample2D, attention_processor.py Attention),
restated with diffusers' module and parameter names so that a real checkpoint's decoder weights load unchanged.  Used by
`from_synthetic` (diffusers is not installed here) and as the unsplit decoder the patch-parallel one is checked against.
The encoder is not restated."""
from __future__ import annotations

import torch
from torch import nn
from torch.nn import functional as F


class _Config(dict):
    """diffusers' FrozenDict: a dict whose keys are also attributes."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e


_BASE = dict(in_channels=3, out_channels=3, up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=(128, 256, 512, 512),
             layers_per_block=2, act_fn="silu", latent_channels=4, norm_num_groups=32)
# stabilityai/stable-diffusion-xl-base-1.0 vae/config.json: overflows in fp16, hence force_upcast
SDXL_VAE = dict(_BASE, sample_size=1024, scaling_factor=0.13025, force_upcast=True)
# CompVis/stable-diffusion-v1-4 vae/config.json: runs in fp16
SD15_VAE = dict(_BASE, sample_size=512, scaling_factor=0.18215, force_upcast=False)

EPS = 1e-6


class DecoderOutput:
    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


class ResnetBlock2D(nn.Module):
    """diffusers ResnetBlock2D with temb_channels=None (no time_emb_proj), eps 1e-6, output_scale_factor 1."""

    def __init__(self, cin, cout, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=EPS)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=EPS)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.nonlinearity = nn.SiLU()
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.fused_norm_act = False      # the patch-parallel decoder turns this on: SiLU runs inside the GroupNorm kernel

    def _norm_act_conv(self, x, norm, conv):
        if self.fused_norm_act and hasattr(conv, "halo_plan") and conv.halo_plan(x) is not None:
            return conv.forward_padded(norm(x, pad_for=conv))          # norm + SiLU + halo rows in one kernel
        h = norm(x)
        if not self.fused_norm_act:
            h = self.nonlinearity(h)
        return conv(h)

    def forward(self, x, temb=None):
        h = self._norm_act_conv(x, self.norm1, self.conv1)
        h = self._norm_act_conv(h, self.norm2, self.conv2)
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Attention(nn.Module):
    """diffusers Attention as UNetMidBlock2D builds it for the VAE: one head of width C, inner GroupNorm, biased q/k/v/out,
    residual_connection, rescale_output_factor 1 (AttnProcessor2_0 on a 4-D input)."""

    def __init__(self, c, groups):
        super().__init__()
        self.heads = 1
        self.group_norm = nn.GroupNorm(groups, c, eps=EPS, affine=True)
        self.to_q = nn.Linear(c, c, bias=True)
        self.to_k = nn.Linear(c, c, bias=True)
        self.to_v = nn.Linear(c, c, bias=True)
        self.to_out = nn.ModuleList([nn.Linear(c, c, bias=True), nn.Dropout(0.0)])
        self.residual_connection = True
        self.rescale_output_factor = 1.0

    def forward(self, x, temb=None):
        residual = x
        b, c, h, w = x.shape
        t = self.group_norm(x.reshape(b, c, h * w)).transpose(1, 2)
        q, k, v = self.to_q(t), self.to_k(t), self.to_v(t)
        o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
        o = self.to_out[1](self.to_out[0](o))
        o = o.transpose(1, 2).reshape(b, c, h, w)
        return (o + residual) / self.rescale_output_factor


class Upsample2D(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class UNetMidBlock2D(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, groups), ResnetBlock2D(c, c, groups)])
        self.attentions = nn.ModuleList([Attention(c, groups)])

    def forward(self, x, temb=None):
        x = self.resnets[0](x)
        for attn, resnet in zip(self.attentions, self.resnets[1:]):
            x = resnet(attn(x))
        return x


class UpDecoderBlock2D(nn.Module):
    def __init__(self, cin, cout, layers, groups, upsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, groups) for i in range(layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if upsample else None

    def forward(self, x, temb=None):
        for resnet in self.resnets:
            x = resnet(x)
        if self.upsamplers is not None:
            for up in self.upsamplers:
                x = up(x)
        return x


class Decoder(nn.Module):
    def __init__(self, in_channels, out_channels, block_out_channels, layers_per_block, norm_num_groups):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = nn.Conv2d(in_channels, rev[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(rev[0], norm_num_groups)
        self.up_blocks = nn.ModuleList()
        out_c = rev[0]
        for i, c in enumerate(rev):
            prev, out_c = out_c, c
            self.up_blocks.append(UpDecoderBlock2D(prev, out_c, layers_per_block + 1, norm_num_groups, i < len(rev) - 1))
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, block_out_channels[0], eps=EPS)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, 3, padding=1)
        self.fused_norm_act = False

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        # diffusers' Decoder.forward: the up blocks run in their own dtype (fp32 under StableDiffusionXLPipeline.upcast_vae(),
        # which leaves conv_in and the mid block in fp16)
        x = x.to(next(iter(self.up_blocks.parameters())).dtype)
        for blk in self.up_blocks:
            x = blk(x)
        if self.fused_norm_act and hasattr(self.conv_out, "halo_plan") and self.conv_out.halo_plan(x) is not None:
            return self.conv_out.forward_padded(self.conv_norm_out(x, pad_for=self.conv_out))
        x = self.conv_norm_out(x)
        if not self.fused_norm_act:
            x = self.conv_act(x)
        return self.conv_out(x)


class AutoencoderKL(nn.Module):
    """The decoding half of diffusers' AutoencoderKL: post_quant_conv + decoder, `decode(z, return_dict)` and `config`."""

    def __init__(self, **config):
        super().__init__()
        cfg = _Config(SD15_VAE)
        cfg.update(config)
        if any(t != "UpDecoderBlock2D" for t in cfg.up_block_types) or cfg.act_fn != "silu":
            raise NotImplementedError("the restated decoder has UpDecoderBlock2D blocks with SiLU only (every SD / SDXL VAE)")
        self.config = cfg
        self.decoder = Decoder(cfg.latent_channels, cfg.out_channels, tuple(cfg.block_out_channels), cfg.layers_per_block,
                               cfg.norm_num_groups)
        self.post_quant_conv = nn.Conv2d(cfg.latent_channels, cfg.latent_channels, 1)

    def decode(self, z, return_dict: bool = True, generator=None):
        """`generator` is unused (diffusers passes it for decoders that sample)."""
        x = self.decoder(self.post_quant_conv(z))
        return DecoderOutput(x) if return_dict else (x,)

    def forward(self, z):
        return self.decode(z).sample
