"""TEST INFRASTRUCTURE (oracle) -- not product code.

CPU restatement of the slice of ``diffusers==0.24.0`` that the reference touches
(reference pins it at /root/reference/setup.py:14; the package is NOT vendored under
/root/reference and is not installed in this image, so this topology is restated from
the published 0.24.0 behaviour: **parity unpinned** at the diffusers boundary -- it is
checkable only by shape and by parameter count: 2 567 463 684 for SDXL, 859 520 964 for
SD1.x, both asserted in tests/test_oracle_unet.py).

It exists so that the UNMODIFIED reference modules
(/root/reference/distrifuser/modules/pp/*.py, models/distri_sdxl_unet_pp.py) can be
imported and executed on CPU (gloo) to generate golden vectors, and so that the oracle's
own restatement of those modules (oracle/pp_modules.py) has a UNet to live in on the GPU
box where /root/reference does not exist.

State-dict keys follow diffusers exactly (``down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q.weight`` ...)
so the product's UNet and this one exchange weights with ``load_state_dict``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from types import SimpleNamespace

import torch
from torch import nn
from torch.nn import functional as F

from .attention import BasicTransformerBlock
from .resnet import Downsample2D, ResnetBlock2D, Upsample2D


@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor = None

    def __getitem__(self, i):
        return (self.sample,)[i]


class ConfigMixin:
    pass


class ModelMixin(nn.Module):
    pass


# --------------------------------------------------------------------------- configs
def sdxl_config() -> dict:
    return dict(
        in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
        up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        transformer_layers_per_block=(1, 2, 10), attention_head_dim=(5, 10, 20),
        cross_attention_dim=2048, use_linear_projection=True, norm_num_groups=32, norm_eps=1e-5,
        addition_embed_type="text_time", addition_time_embed_dim=256,
        projection_class_embeddings_input_dim=2816,
    )


def sd15_config() -> dict:
    return dict(
        in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
        down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
        up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3,
        transformer_layers_per_block=(1, 1, 1, 1), attention_head_dim=(8, 8, 8, 8),
        cross_attention_dim=768, use_linear_projection=False, norm_num_groups=32, norm_eps=1e-5,
        addition_embed_type=None, addition_time_embed_dim=None,
        projection_class_embeddings_input_dim=None,
    )


def tiny_sdxl_config() -> dict:
    """SDXL topology at 1/5 width (head_dim stays 64) -- parity-test workload."""
    cfg = sdxl_config()
    cfg.update(block_out_channels=(64, 128, 256), transformer_layers_per_block=(1, 1, 2),
               attention_head_dim=(1, 2, 4), cross_attention_dim=64,
               addition_time_embed_dim=32, projection_class_embeddings_input_dim=32 * 6 + 48)
    return cfg


def tiny_sd15_config() -> dict:
    """SD1.x topology, narrow: head dims 40/80/160/160 like the real one (8 heads -> 2 heads)."""
    cfg = sd15_config()
    cfg.update(block_out_channels=(80, 160, 320, 320), attention_head_dim=(2, 2, 2, 2),
               cross_attention_dim=48, norm_num_groups=8)
    return cfg


# --------------------------------------------------------------------------- embeddings
def get_timestep_embedding(timesteps, dim, flip_sin_to_cos=True, downscale_freq_shift=0.0, max_period=10000):
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=timesteps.device)
    exponent = exponent / (half - downscale_freq_shift)
    emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return emb


class Timesteps(nn.Module):
    def __init__(self, num_channels, flip_sin_to_cos=True, downscale_freq_shift=0.0):
        super().__init__()
        self.num_channels, self.flip, self.shift = num_channels, flip_sin_to_cos, downscale_freq_shift

    def forward(self, t):
        return get_timestep_embedding(t, self.num_channels, self.flip, self.shift)


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels, time_embed_dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, x):
        return self.linear_2(self.act(self.linear_1(x)))


def embed(model, sample, timestep, added_cond_kwargs):
    """Time embedding of a UNet or ControlNet call, plus SDXL's added (text_time) embedding: emb [B, temb]."""
    timesteps = timestep
    if not torch.is_tensor(timesteps):
        timesteps = torch.tensor([timesteps], dtype=torch.int64, device=sample.device)
    elif timesteps.ndim == 0:
        timesteps = timesteps[None].to(sample.device)
    timesteps = timesteps.expand(sample.shape[0])
    emb = model.time_embedding(model.time_proj(timesteps).to(sample.dtype))
    if model.config.addition_embed_type == "text_time":
        text_embeds = added_cond_kwargs["text_embeds"]
        time_ids = added_cond_kwargs["time_ids"]
        time_embeds = model.add_time_proj(time_ids.flatten()).reshape(text_embeds.shape[0], -1)
        add = torch.cat([text_embeds, time_embeds], dim=-1).to(emb.dtype)
        emb = emb + model.add_embedding(add)
    return emb


# --------------------------------------------------------------------------- transformer
class Transformer2DModel(nn.Module):
    def __init__(self, heads, head_dim, in_channels, depth, cross_dim, groups, use_linear_projection):
        super().__init__()
        inner = heads * head_dim
        self.use_linear_projection = use_linear_projection
        self.norm = nn.GroupNorm(groups, in_channels, eps=1e-6, affine=True)
        if use_linear_projection:
            self.proj_in = nn.Linear(in_channels, inner)
        else:
            self.proj_in = nn.Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner, heads, head_dim, cross_dim) for _ in range(depth)])
        if use_linear_projection:
            self.proj_out = nn.Linear(inner, in_channels)
        else:
            self.proj_out = nn.Conv2d(inner, in_channels, 1)

    def forward(self, hidden_states, encoder_hidden_states=None):
        b, _, h, w = hidden_states.shape
        residual = hidden_states
        hidden_states = self.norm(hidden_states)
        if self.use_linear_projection:
            inner = hidden_states.shape[1]
            hidden_states = hidden_states.permute(0, 2, 3, 1).reshape(b, h * w, inner)
            hidden_states = self.proj_in(hidden_states)
        else:
            hidden_states = self.proj_in(hidden_states)
            inner = hidden_states.shape[1]
            hidden_states = hidden_states.permute(0, 2, 3, 1).reshape(b, h * w, inner)
        for block in self.transformer_blocks:
            hidden_states = block(hidden_states, encoder_hidden_states=encoder_hidden_states)
        if self.use_linear_projection:
            hidden_states = self.proj_out(hidden_states)
            hidden_states = hidden_states.reshape(b, h, w, inner).permute(0, 3, 1, 2).contiguous()
        else:
            hidden_states = hidden_states.reshape(b, h, w, inner).permute(0, 3, 1, 2).contiguous()
            hidden_states = self.proj_out(hidden_states)
        return hidden_states + residual


# --------------------------------------------------------------------------- blocks
class DownBlock2D(nn.Module):
    has_cross_attention = False

    def __init__(self, cin, cout, temb, layers, groups, eps, add_downsample, **_):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, h, temb, encoder_hidden_states=None):
        out = ()
        for resnet in self.resnets:
            h = resnet(h, temb)
            out += (h,)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                h = d(h)
            out += (h,)
        return h, out


class CrossAttnDownBlock2D(nn.Module):
    has_cross_attention = True

    def __init__(self, cin, cout, temb, layers, groups, eps, add_downsample, heads, depth, cross_dim, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList(
            [ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(layers)])
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, depth, cross_dim, groups, linear_proj)
             for _ in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, h, temb, encoder_hidden_states=None):
        out = ()
        for resnet, attn in zip(self.resnets, self.attentions):
            h = resnet(h, temb)
            h = attn(h, encoder_hidden_states=encoder_hidden_states)
            out += (h,)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                h = d(h)
            out += (h,)
        return h, out


class UNetMidBlock2DCrossAttn(nn.Module):
    def __init__(self, c, temb, groups, eps, heads, depth, cross_dim, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, groups, eps), ResnetBlock2D(c, c, temb, groups, eps)])
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, c // heads, c, depth, cross_dim, groups, linear_proj)])

    def forward(self, h, temb, encoder_hidden_states=None):
        h = self.resnets[0](h, temb)
        for attn, resnet in zip(self.attentions, self.resnets[1:]):
            h = attn(h, encoder_hidden_states=encoder_hidden_states)
            h = resnet(h, temb)
        return h


class UpBlock2D(nn.Module):
    has_cross_attention = False

    def __init__(self, cin, cout, prev, temb, layers, groups, eps, add_upsample, **_):
        super().__init__()
        resnets = []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            rin = prev if i == 0 else cout
            resnets.append(ResnetBlock2D(rin + skip, cout, temb, groups, eps))
        self.resnets = nn.ModuleList(resnets)
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, h, res_tuple, temb, encoder_hidden_states=None):
        for resnet in self.resnets:
            res = res_tuple[-1]
            res_tuple = res_tuple[:-1]
            h = torch.cat([h, res], dim=1)
            h = resnet(h, temb)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                h = u(h)
        return h


class CrossAttnUpBlock2D(nn.Module):
    has_cross_attention = True

    def __init__(self, cin, cout, prev, temb, layers, groups, eps, add_upsample, heads, depth, cross_dim, linear_proj):
        super().__init__()
        resnets, attns = [], []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            rin = prev if i == 0 else cout
            resnets.append(ResnetBlock2D(rin + skip, cout, temb, groups, eps))
            attns.append(Transformer2DModel(heads, cout // heads, cout, depth, cross_dim, groups, linear_proj))
        self.resnets = nn.ModuleList(resnets)
        self.attentions = nn.ModuleList(attns)
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, h, res_tuple, temb, encoder_hidden_states=None):
        for resnet, attn in zip(self.resnets, self.attentions):
            res = res_tuple[-1]
            res_tuple = res_tuple[:-1]
            h = torch.cat([h, res], dim=1)
            h = resnet(h, temb)
            h = attn(h, encoder_hidden_states=encoder_hidden_states)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                h = u(h)
        return h


# --------------------------------------------------------------------------- UNet
class UNet2DConditionModel(ModelMixin, ConfigMixin):
    """Topology of diffusers-0.24.0 ``UNet2DConditionModel`` for the SD1.x / SDXL configs."""

    def __init__(self, **cfg):
        super().__init__()
        full = sdxl_config()
        full.update(cfg)
        self.config = SimpleNamespace(**full)
        c = self.config
        boc = tuple(c.block_out_channels)
        temb = boc[0] * 4
        g, eps = c.norm_num_groups, c.norm_eps
        self.conv_in = nn.Conv2d(c.in_channels, boc[0], 3, padding=1)
        self.time_proj = Timesteps(boc[0], True, 0)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        if c.addition_embed_type == "text_time":
            self.add_time_proj = Timesteps(c.addition_time_embed_dim, True, 0)
            self.add_embedding = TimestepEmbedding(c.projection_class_embeddings_input_dim, temb)
        nb = len(boc)
        heads, depth = tuple(c.attention_head_dim), tuple(c.transformer_layers_per_block)
        self.down_blocks = nn.ModuleList()
        out_ch = boc[0]
        for i, t in enumerate(c.down_block_types):
            in_ch, out_ch = out_ch, boc[i]
            cls = CrossAttnDownBlock2D if t == "CrossAttnDownBlock2D" else DownBlock2D
            self.down_blocks.append(cls(in_ch, out_ch, temb, c.layers_per_block, g, eps, i != nb - 1,
                                        heads=heads[i], depth=depth[i], cross_dim=c.cross_attention_dim,
                                        linear_proj=c.use_linear_projection))
        self.mid_block = UNetMidBlock2DCrossAttn(boc[-1], temb, g, eps, heads[-1], depth[-1],
                                                 c.cross_attention_dim, c.use_linear_projection)
        self.up_blocks = nn.ModuleList()
        rboc, rheads, rdepth = boc[::-1], heads[::-1], depth[::-1]
        out_ch = rboc[0]
        for i, t in enumerate(c.up_block_types):
            prev, out_ch = out_ch, rboc[i]
            in_ch = rboc[min(i + 1, nb - 1)]
            cls = CrossAttnUpBlock2D if t == "CrossAttnUpBlock2D" else UpBlock2D
            self.up_blocks.append(cls(in_ch, out_ch, prev, temb, c.layers_per_block + 1, g, eps, i != nb - 1,
                                      heads=rheads[i], depth=rdepth[i], cross_dim=c.cross_attention_dim,
                                      linear_proj=c.use_linear_projection))
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=eps)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(boc[0], c.out_channels, 3, padding=1)

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs=None, added_cond_kwargs=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None,
                down_intrablock_additional_residuals=None, encoder_attention_mask=None, return_dict=True):
        emb = embed(self, sample, timestep, added_cond_kwargs)
        sample = self.conv_in(sample)
        res = (sample,)
        for blk in self.down_blocks:
            sample, out = blk(sample, emb, encoder_hidden_states=encoder_hidden_states)
            res += out
        if down_block_additional_residuals is not None:      # ControlNet: skip i + residual i
            res = tuple(r + d for r, d in zip(res, down_block_additional_residuals, strict=True))
        sample = self.mid_block(sample, emb, encoder_hidden_states=encoder_hidden_states)
        if mid_block_additional_residual is not None:
            sample = sample + mid_block_additional_residual
        for blk in self.up_blocks:
            n = len(blk.resnets)
            r, res = res[-n:], res[:-n]
            sample = blk(sample, r, emb, encoder_hidden_states=encoder_hidden_states)
        sample = self.conv_out(self.conv_act(self.conv_norm_out(sample)))
        if not return_dict:
            return (sample,)
        return UNet2DConditionOutput(sample=sample)
