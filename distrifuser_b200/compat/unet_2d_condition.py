"""UNet2DConditionModel for environments without `diffusers` (this image has none and no network).

The reference pins diffusers==0.24.0 (setup.py:14) and wraps its UNet2DConditionModel
(distrifuser/models/distri_sdxl_unet_pp.py:16-40).  This module provides the same module tree -- attribute names,
call signatures and state-dict keys of the SD1.x / SDXL configurations -- so that DistriUNetPP's surgery and
real checkpoints work unchanged, and `DistriSDXLPipeline.from_pretrained` uses the real diffusers class when it
is importable.  Activations are kept NHWC (torch.channels_last) end to end: the [b,C,h,w] <-> [b,hw,C] reshapes
around the transformer blocks are then free views and cuDNN gets tensor-core friendly layouts.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch
from torch import nn
from torch.nn import functional as F

SDXL = dict(
    in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
    down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
    up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
    transformer_layers_per_block=(1, 2, 10), attention_head_dim=(5, 10, 20), cross_attention_dim=2048,
    use_linear_projection=True, norm_num_groups=32, norm_eps=1e-5, addition_embed_type="text_time",
    addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816, sample_size=128,
)
SD15 = dict(
    in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
    down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
    up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3,
    transformer_layers_per_block=(1, 1, 1, 1), attention_head_dim=(8, 8, 8, 8), cross_attention_dim=768,
    use_linear_projection=False, norm_num_groups=32, norm_eps=1e-5, addition_embed_type=None,
    addition_time_embed_dim=None, projection_class_embeddings_input_dim=None, sample_size=64,
)


class UNet2DConditionOutput:
    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


class Attention(nn.Module):
    """Attribute contract read by DistriAttentionPP (attn.py:16-38,93-100)."""

    def __init__(self, query_dim, cross_attention_dim, heads, dim_head):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.inner_dim = heads, inner
        self.residual_connection, self.rescale_output_factor = False, 1.0
        kv_dim = query_dim if cross_attention_dim is None else cross_attention_dim
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(kv_dim, inner, bias=False)
        self.to_v = nn.Linear(kv_dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])

    def forward(self, hidden_states, encoder_hidden_states=None, **kw):
        raise RuntimeError("Attention must be wrapped by DistriSelfAttentionPP / DistriCrossAttentionPP "
                           "(distrifuser_b200 has no unfused attention path)")


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)
        self._fused = None            # (key, interleaved weight, interleaved bias) of the one-kernel projection + gate
        self.norm_fused = None        # set by BasicTransformerBlock: LayerNorm whose output feeds this projection (unused here)

    def _fused_weights(self, block):
        """Interleaved copy of proj.weight / proj.bias for the fused wgmma GEMM + GEGLU epilogue (ops.linear_geglu); rebuilt
        when the source tensors change (load_state_dict, .to(), in-place edits) or the kernel wants another block size."""
        from .. import ops
        w, b = self.proj.weight, self.proj.bias
        key = (block, w._version, w.data_ptr(), w.dtype, w.device, None if b is None else (b._version, b.data_ptr()))
        if self._fused is None or self._fused[0] != key:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("GEGLU: weights changed since the last eager call; run one eager UNet call before capturing graphs")
            with torch.no_grad():
                wi, bi = ops.geglu_interleave(w.detach(), None if b is None else b.detach(), block)
            self._fused = (key, wi, bi)
        return self._fused[1], self._fused[2]

    def forward(self, x):
        if x.is_cuda and x.dtype == torch.float16:
            from .. import ops
            D, K = self.proj.out_features // 2, self.proj.in_features
            block = ops.geglu_block(x.numel() // K, 2 * D, K) if ops.use_fused_linear("geglu") else 0
            if block:
                wi, bi = self._fused_weights(block)
                return ops.linear_geglu(x, wi, bi, block)   # projection + gate in ONE kernel: the [.., 8C] tensor never exists
            return ops.geglu(self.proj(x))                  # library GEMM + one fused gate kernel
        y = self.proj(x)
        x, gate = y.chunk(2, dim=-1)
        return x * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, 4 * dim), nn.Dropout(0.0), nn.Linear(4 * dim, dim)])

    def forward(self, x):
        from .. import ops
        return ops.project("ff2", self.net[0](x), self.net[2])


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, head_dim, cross_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, head_dim)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_dim, heads, head_dim)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)

    def forward_chained(self, x, pending, encoder_hidden_states=None):
        """Fused path: the block input is `x + pending` (pending = the previous block's feed-forward output, or None); returns
        (x', pending') with the true output x' + pending', so that the trailing residual add is fused into the next block's
        first add+LayerNorm kernel."""
        from ..ops import add_layernorm              # residual add + LayerNorm in one kernel
        x, h = add_layernorm(x, pending, self.norm1)
        x, h = add_layernorm(x, self.attn1(h, encoder_hidden_states=None), self.norm2)
        x, h = add_layernorm(x, self.attn2(h, encoder_hidden_states=encoder_hidden_states), self.norm3)
        return x, self.ff(h)

    def forward(self, x, encoder_hidden_states=None):
        if x.is_cuda and x.dtype == torch.float16:
            x, pending = self.forward_chained(x, None, encoder_hidden_states)
            return x + pending
        x = x + self.attn1(self.norm1(x), encoder_hidden_states=None)
        x = x + self.attn2(self.norm2(x), encoder_hidden_states=encoder_hidden_states)
        return x + self.ff(self.norm3(x))


class Transformer2DModel(nn.Module):
    def __init__(self, heads, head_dim, channels, depth, cross_dim, groups, linear_proj):
        super().__init__()
        inner = heads * head_dim
        self.use_linear_projection = linear_proj
        self.norm = nn.GroupNorm(groups, channels, eps=1e-6)
        self.proj_in = nn.Linear(channels, inner) if linear_proj else nn.Conv2d(channels, inner, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, head_dim, cross_dim) for _ in range(depth)])
        self.proj_out = nn.Linear(inner, channels) if linear_proj else nn.Conv2d(inner, channels, 1)

    @staticmethod
    def _tokens(x):  # [b,C,h,w] (NHWC memory) -> [b,hw,C] without a copy
        b, c, h, w = x.shape
        return x.permute(0, 2, 3, 1).reshape(b, h * w, c)

    @staticmethod
    def _image(t, h, w):  # [b,hw,C] -> [b,C,h,w] NHWC memory, no copy
        b, _, c = t.shape
        return t.reshape(b, h, w, c).permute(0, 3, 1, 2)

    def forward(self, x, encoder_hidden_states=None):
        _, _, h, w = x.shape
        res = x
        x = self.norm(x)
        if self.use_linear_projection:
            from .. import ops
            t = ops.project("proj", self._tokens(x), self.proj_in)
        else:
            t = self._tokens(self.proj_in(x))
        if t.is_cuda and t.dtype == torch.float16:
            pending = None
            for blk in self.transformer_blocks:
                t, pending = blk.forward_chained(t, pending, encoder_hidden_states)
            t = t + pending
        else:
            for blk in self.transformer_blocks:
                t = blk(t, encoder_hidden_states=encoder_hidden_states)
        if self.use_linear_projection:
            x = self._image(ops.project("proj", t, self.proj_out), h, w)
        else:
            x = self.proj_out(self._image(t, h, w))
        return x + res


class ResnetBlock2D(nn.Module):
    def __init__(self, cin, cout, temb, groups, eps):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb, cout)
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.nonlinearity = nn.SiLU()
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.output_scale_factor = 1.0
        self.fused_norm_act = False      # DistriUNetPP turns this on: SiLU runs inside the GroupNorm kernel
        self.temb_proj = None            # [b, cout] view set by the UNet per call: time_emb_proj(silu(temb)) of ALL blocks in one GEMM
        self.temb_has_conv1_bias = False # ... which then already contains conv1.bias (conv1 runs without its bias pass)

    def folds_conv1_bias(self) -> bool:
        return self.fused_norm_act and _conv_of(self.conv1).bias is not None

    def _tail_bias(self):
        """conv2.bias + conv_shortcut.bias as one vector (cached on the parameters' versions): added together with the
        residual in ONE pass after conv2 (ops.conv2d_bias_residual)."""
        c2 = _conv_of(self.conv2)
        if self.conv_shortcut is None or self.conv_shortcut.bias is None:
            return c2.bias
        key = (c2.bias._version, self.conv_shortcut.bias._version, c2.bias.data_ptr())
        cache = getattr(self, "_tail_bias_cache", None)
        if cache is None or cache[0] != key:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("conv biases changed since the last eager call; run one eager UNet call before capture")
            with torch.no_grad():
                self._tail_bias_cache = cache = (key, (c2.bias.detach() + self.conv_shortcut.bias.detach()).contiguous())
        return cache[1]

    def forward(self, x, temb):
        fused_halo = self.fused_norm_act and hasattr(self.conv1, "halo_plan")    # DistriGroupNorm -> DistriConv2dPP pairs
        fold1 = self.temb_proj is not None and self.temb_has_conv1_bias          # conv1.bias is inside temb_proj
        fused_tail = self.fused_norm_act and hasattr(self.conv2, "halo_plan") and x.is_cuda and x.dtype == torch.float16
        k1 = dict(fold_bias=True) if fold1 else {}
        if fused_halo and self.conv1.halo_plan(x) is not None:
            h = self.conv1.forward_padded(self.norm1(x, pad_for=self.conv1), **k1)     # norm + SiLU + halo rows in ONE kernel
        else:
            h = self.norm1(x)
            if not self.fused_norm_act:
                h = self.nonlinearity(h)
            h = self.conv1(h, **k1)
        t = self.temb_proj if self.temb_proj is not None else self.time_emb_proj(self.nonlinearity(temb))
        if fused_tail:
            # shortcut without its bias pass; conv2 without bias; then conv2.bias + shortcut.bias + residual in one pass
            sc = self.conv_shortcut
            res = x if sc is None else F.conv2d(x, sc.weight)
            tail_bias = self._tail_bias()
            if fused_halo and self.conv2.halo_plan(h) is not None:
                return self.conv2.forward_padded(self.norm2(h, addend=t, pad_for=self.conv2), residual=res, bias=tail_bias)
            return self.conv2(self.norm2(h, addend=t), residual=res, bias=tail_bias)
        if fused_halo and self.conv2.halo_plan(h) is not None:
            h = self.conv2.forward_padded(self.norm2(h, addend=t, pad_for=self.conv2))
        else:
            if self.fused_norm_act:
                h = self.norm2(h, addend=t)      # GroupNorm(h + t[:, :, None, None]) + SiLU in one kernel
            else:
                h = self.nonlinearity(self.norm2(h + t[:, :, None, None]))
            h = self.conv2(h)
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


def _conv_of(m):
    """the nn.Conv2d behind a DistriConv2dPP wrapper (or the module itself)."""
    return m.module if hasattr(m, "module") and isinstance(getattr(m, "module"), nn.Conv2d) else m


class Downsample2D(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class _Down(nn.Module):
    def __init__(self, cin, cout, temb, layers, groups, eps, downsample, attn):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(layers)])
        if attn is not None:
            self.attentions = nn.ModuleList([Transformer2DModel(channels=cout, groups=groups, **attn) for _ in range(layers)])
        self.has_cross_attention = attn is not None
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if downsample else None

    def forward(self, x, temb, ehs):
        skips = []
        for i, res in enumerate(self.resnets):
            x = res(x, temb)
            if self.has_cross_attention:
                x = self.attentions[i](x, encoder_hidden_states=ehs)
            skips.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            skips.append(x)
        return x, skips


class _Mid(nn.Module):
    def __init__(self, c, temb, groups, eps, attn):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([Transformer2DModel(channels=c, groups=groups, **attn)])

    def forward(self, x, temb, ehs):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, encoder_hidden_states=ehs)
        return self.resnets[1](x, temb)


class _Up(nn.Module):
    def __init__(self, cin, cout, prev, temb, layers, groups, eps, upsample, attn):
        super().__init__()
        self.resnets = nn.ModuleList()
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            self.resnets.append(ResnetBlock2D((prev if i == 0 else cout) + skip, cout, temb, groups, eps))
        if attn is not None:
            self.attentions = nn.ModuleList([Transformer2DModel(channels=cout, groups=groups, **attn) for _ in range(layers)])
        self.has_cross_attention = attn is not None
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if upsample else None

    def forward(self, x, skips, temb, ehs):
        for i, res in enumerate(self.resnets):
            x = res(torch.cat([x, skips.pop()], dim=1), temb)
            if self.has_cross_attention:
                x = self.attentions[i](x, encoder_hidden_states=ehs)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class TimestepEmbedding(nn.Module):
    def __init__(self, cin, dim):
        super().__init__()
        self.linear_1 = nn.Linear(cin, dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(self.act(self.linear_1(x)))


def sinusoid(t: torch.Tensor, dim: int) -> torch.Tensor:
    """diffusers Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0): [cos | sin]."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    ang = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(ang), torch.sin(ang)], dim=-1)


def embed(model, sample, timestep, added_cond_kwargs):
    """Time embedding of a UNet or ControlNet call plus SDXL's added (text_time) embedding -> emb [B, temb]; also hands every
    ResnetBlock2D its projection of emb (model._batched_temb)."""
    c = model.config
    t = timestep
    if not torch.is_tensor(t):
        t = torch.tensor([t], dtype=torch.float32, device=sample.device)
    elif t.ndim == 0:
        t = t[None]
    t = t.to(sample.device).expand(sample.shape[0])
    emb = model.time_embedding(sinusoid(t, c.block_out_channels[0]).to(sample.dtype))
    if c.addition_embed_type == "text_time":
        text, ids = added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"]
        tid = sinusoid(ids.flatten(), c.addition_time_embed_dim).reshape(text.shape[0], -1)
        emb = emb + model.add_embedding(torch.cat([text, tid.to(text.dtype)], dim=-1).to(emb.dtype))
    model._batched_temb(emb)
    return emb


class UNet2DConditionModel(nn.Module):
    def __init__(self, **overrides):
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
        self.down_blocks = nn.ModuleList()
        ch = boc[0]
        for i, kind in enumerate(c.down_block_types):
            cin, ch = ch, boc[i]
            self.down_blocks.append(_Down(cin, ch, temb, c.layers_per_block, g, eps, i != nb - 1,
                                          attn_cfg(i, ch) if kind.startswith("CrossAttn") else None))
        self.mid_block = _Mid(boc[-1], temb, g, eps, attn_cfg(nb - 1, boc[-1]))
        self.up_blocks = nn.ModuleList()
        rev = boc[::-1]
        ch = rev[0]
        for i, kind in enumerate(c.up_block_types):
            prev, ch = ch, rev[i]
            cin = rev[min(i + 1, nb - 1)]
            self.up_blocks.append(_Up(cin, ch, prev, temb, c.layers_per_block + 1, g, eps, i != nb - 1,
                                      attn_cfg(nb - 1 - i, ch) if kind.startswith("CrossAttn") else None))
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=eps)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(boc[0], c.out_channels, 3, padding=1)
        self.fused_norm_act = False

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    def _resnets(self):
        return [m for m in self.modules() if isinstance(m, ResnetBlock2D)]

    def _batched_temb(self, emb):
        """time_emb_proj(silu(emb)) of every ResnetBlock2D as ONE GEMM + one SiLU per UNet call instead of 17 tiny pairs (the
        activation function and the embedding are the same for all blocks); the concatenated weight follows the blocks' weights
        (version counters).  Sets blk.temb_proj views; a no-op on CPU / non-fp16 (reference path of the tests)."""
        blocks = self._resnets()
        if not (emb.is_cuda and emb.dtype == torch.float16) or not blocks:
            for blk in blocks:
                blk.temb_proj = None
                blk.temb_has_conv1_bias = False
            return
        fold = [blk.folds_conv1_bias() for blk in blocks]
        key = tuple((blk.time_emb_proj.weight._version, blk.time_emb_proj.weight.data_ptr(), blk.time_emb_proj.bias._version,
                     _conv_of(blk.conv1).bias._version if f else -1) for blk, f in zip(blocks, fold))
        cache = getattr(self, "_temb_cache", None)
        if cache is None or cache[0] != key:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("time-embedding weights changed since the last eager call; run one eager UNet call before capture")
            with torch.no_grad():
                w = torch.cat([blk.time_emb_proj.weight.detach() for blk in blocks], 0).contiguous()
                # conv1.bias rides on the embedding: GroupNorm(conv1(x) + b1 + t) == GroupNorm(conv1(x) + (t + b1)), so conv1
                # runs without its bias pass (ResnetBlock2D.forward, fused path)
                b = torch.cat([blk.time_emb_proj.bias.detach() + (_conv_of(blk.conv1).bias.detach() if f else 0)
                               for blk, f in zip(blocks, fold)], 0).contiguous()
            self._temb_cache = cache = (key, w, b)
        allp = F.linear(F.silu(emb), cache[1], cache[2])
        o = 0
        for blk, f in zip(blocks, fold):
            n = blk.time_emb_proj.out_features
            blk.temb_proj = allp[:, o:o + n]
            blk.temb_has_conv1_bias = f
            o += n

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None, attention_mask=None,
                cross_attention_kwargs=None, added_cond_kwargs=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, down_intrablock_additional_residuals=None,
                encoder_attention_mask=None, return_dict=True):
        emb = embed(self, sample, timestep, added_cond_kwargs)
        x = self.conv_in(sample)
        skips = [x]
        for blk in self.down_blocks:
            x, s = blk(x, emb, encoder_hidden_states)
            skips += s
        if down_block_additional_residuals is not None:              # ControlNet: skip i + residual i, as diffusers adds them
            skips = [s + r for s, r in zip(skips, down_block_additional_residuals, strict=True)]
        x = self.mid_block(x, emb, encoder_hidden_states)
        if mid_block_additional_residual is not None:
            x = x + mid_block_additional_residual
        for blk in self.up_blocks:
            x = blk(x, skips, emb, encoder_hidden_states)
        if self.fused_norm_act and hasattr(self.conv_out, "halo_plan") and self.conv_out.halo_plan(x) is not None:
            x = self.conv_out.forward_padded(self.conv_norm_out(x, pad_for=self.conv_out))
        else:
            x = self.conv_norm_out(x)
            if not self.fused_norm_act:
                x = self.conv_act(x)
            x = self.conv_out(x)
        return UNet2DConditionOutput(x) if return_dict else (x,)
