"""DistriAutoencoderKLPP -- the VAE decode split over every GPU of the world by latent rows (patch parallelism for the decoder).

At decode time every rank holds the same final latents, so every world rank takes part (no CFG split): the wrappers see a
world-wide view of the config (n_device_per_batch = world_size, split_idx = rank, mode "full_sync"), and rank r decodes the
image rows of latent rows split_units(h, n)[r].  Every exchange is synchronous, so the split decode equals the one-device
decode up to fp16 rounding:
  * 3x3 convs: halo rows from the strip neighbours (DistriConv2dPP), fused into the GroupNorm that feeds the conv where one
    does, and by push + assemble after the nearest upsamplers; the decoder's conv_in slices its rows from the whole latent;
  * GroupNorm: the moments of the whole image, each rank's weighted by its rows, with nn.GroupNorm's biased variance;
  * mid-block attention: every rank's K/V segment through the arena, df_attn_wide_fwd (DistriVAEAttentionPP);
  * the [B, 3, 8h, 8w] image: df_output_gather_2d, which is also the per-call world barrier the arena's banks rely on
    (BANK-REUSE INVARIANT, utils.py).
The decoder has its own PatchParallelismCommManager (arena, flags, epoch clock), so the UNet's arena is untouched.

upcast=True decodes a VAE that overflows fp16 (force_upcast, e.g. the stock SDXL VAE) with the precision split of diffusers'
StableDiffusionXLPipeline.upcast_vae(): post_quant_conv, conv_in and the mid block (with its attention) in fp16, the up blocks,
conv_norm_out and conv_out in fp32.  The GroupNorm, halo and gather kernels then run their fp32 instantiations there."""
import copy

import torch
from torch import distributed as dist
from torch import nn

from .. import _lib
from ..compat.vae import DecoderOutput
from ..modules.base_module import BaseModule
from ..modules.pp.conv2d import DistriConv2dPP
from ..modules.pp.groupnorm import DistriGroupNorm
from ..modules.pp.vae_attn import DistriVAEAttentionPP
from ..utils import DistriConfig, PatchParallelismCommManager, row_offset, split_units


def _is_vae_attention(m: nn.Module) -> bool:
    return all(hasattr(m, a) for a in ("to_q", "to_k", "to_v", "to_out", "group_norm"))


# the decoder's parts that diffusers' upcast_vae() leaves in fp32 (everything after the mid block)
UPCAST_PARTS = ("up_blocks", "conv_norm_out", "conv_out")


def install_vae_wrappers(decoder: nn.Module, distri_config: DistriConfig, upcast: bool = False) -> None:
    """Module surgery of the decoder in place: 3x3 convs, GroupNorms (biased variance) and the mid-block attention become the
    sm_90a wrappers, GroupNorm -> SiLU pairs fuse, and the decoder goes channels_last.  upcast: the wrappers of UPCAST_PARTS
    take fp32 tensors."""
    for _, module in list(decoder.named_modules()):
        if isinstance(module, BaseModule) or _is_vae_attention(module):
            continue
        for subname, sub in list(module.named_children()):
            if isinstance(sub, nn.Conv2d):
                if tuple(sub.kernel_size) == (1, 1):
                    continue
                setattr(module, subname, DistriConv2dPP(sub, distri_config, is_first_layer=subname == "conv_in"))
            elif _is_vae_attention(sub):
                setattr(module, subname, DistriVAEAttentionPP(sub, distri_config))
            elif isinstance(sub, nn.GroupNorm):
                gn = DistriGroupNorm(sub, distri_config)
                gn.biased_var = True
                setattr(module, subname, gn)
    for module in decoder.modules():
        if hasattr(module, "fused_norm_act"):
            module.fused_norm_act = True
            for nm in ("norm1", "norm2", "conv_norm_out"):
                sub = getattr(module, nm, None)
                if isinstance(sub, DistriGroupNorm):
                    sub.fuse_silu = True
    if upcast:
        for part in UPCAST_PARTS:
            for module in getattr(decoder, part).modules():
                if isinstance(module, BaseModule):
                    module.allow_fp32 = True
    decoder.to(memory_format=torch.channels_last)


def apply_upcast_split(vae: nn.Module) -> None:
    """diffusers' upcast_vae() precision split, whatever the VAE's dtype: the decoder's UPCAST_PARTS in fp32, post_quant_conv,
    conv_in and the mid block in fp16."""
    for m in (vae.post_quant_conv, vae.decoder.conv_in, vae.decoder.mid_block):
        m.to(torch.float16)
    for part in UPCAST_PARTS:
        getattr(vae.decoder, part).to(torch.float32)


def vae_row_plan(latent_rows: int, world: int) -> list[int]:
    """Latent rows of each rank (units of u = 1 row): rank r of n holds h // n or h // n + 1 consecutive rows."""
    if latent_rows < world:
        raise ValueError(f"the patch-parallel VAE decode over {world} ranks needs at least one latent row per rank: the latent "
                         f"has {latent_rows} rows")
    return split_units(latent_rows, world)


class DistriAutoencoderKLPP(nn.Module):
    """Wraps an AutoencoderKL (compat.vae or diffusers) for decoding on every rank; `decode(z, return_dict=True)` and
    `config` as diffusers' AutoencoderKL, so a diffusers pipeline's own `self.vae.decode(...)` runs it.

    upcast=False: the decode runs in fp16 and returns fp16; a VAE whose config sets force_upcast is refused.
    upcast=True: any VAE, with diffusers' precision split (module docstring); decode() takes fp16 latents and returns an fp32
    image.  `config` then reports force_upcast=False (a copy: the VAE's own config is left alone) and `dtype` is fp16, so a
    diffusers SDXL pipeline passes its fp16 latents straight to decode() instead of calling upcast_vae() on the wrapper."""

    def __init__(self, vae: nn.Module, distri_config: DistriConfig, upcast: bool = False):
        super().__init__()
        if not upcast and bool(vae.config.get("force_upcast", False)):
            raise ValueError("this VAE's config sets force_upcast=True: it overflows in fp16 (the stock SDXL VAE does), and "
                             "the patch-parallel decode runs in fp16 unless upcast=True is passed (vae_upcast=True in the "
                             "pipelines), which runs the up blocks in fp32 as diffusers does.  Otherwise use an fp16-safe VAE "
                             "(SD1.x's, or an fp16-fixed SDXL VAE), or set force_upcast=False in its config at your own risk.")
        view = copy.copy(distri_config)
        view.n_device_per_batch = distri_config.world_size       # split_idx() == rank: every world rank is a patch rank
        view.split_batch = False                                 # one patch group: the whole world
        view.mode = "full_sync"
        self.vae = vae
        self.view = view
        self.distri_config = distri_config
        self.upcast = upcast
        self._config = vae.config
        if upcast:
            apply_upcast_split(vae)
            self._config = type(vae.config)({**vae.config, "force_upcast": False})
        install_vae_wrappers(vae.decoder, view, upcast=upcast)
        self.comm_manager = None
        self.row_units = None
        self._layout_key = None
        self.output_buffer = None

    @property
    def config(self):
        return self._config

    @property
    def dtype(self):
        return self.vae.post_quant_conv.weight.dtype

    @property
    def device(self):
        return self.vae.post_quant_conv.weight.device

    def _modules_pp(self):
        return [m for m in self.vae.decoder.modules() if isinstance(m, BaseModule)]

    def _decode_strip(self, z):
        z = self.vae.post_quant_conv(z).contiguous(memory_format=torch.channels_last)
        return self.vae.decoder(z)

    def _out_dtype(self):
        return next(self.vae.decoder.conv_out.parameters()).dtype

    def _lay_out(self, z):
        """Row plan, and with more than one rank the decoder's comm manager, for latents of z's shape: one registration pass
        (the wrappers size their slots by the dtypes they see; its image is discarded), then the arena.  A new shape, upcast
        state or output dtype replaces the previous arena."""
        cfg = self.view
        n = cfg.n_device_per_batch
        b, _, h, w = z.shape
        self.row_units = vae_row_plan(h, n) if n > 1 else None
        modules = self._modules_pp()
        for m in modules:
            m.row_units = self.row_units
        if n == 1:
            return
        if self.comm_manager is not None:
            dist.barrier()                       # every rank is past its last read of the old arenas
            self.comm_manager.close()
            self.comm_manager = None
        for m in modules:
            m.idx = None                         # register again, in the new manager
            m.set_counter(0)
            if isinstance(m, DistriVAEAttentionPP):
                m._kvmaps = None                 # tensor maps of the old arena
        self.output_buffer = None
        cm = PatchParallelismCommManager(cfg)
        cm.register_output(b, self.vae.config.out_channels, 8 * h, 8 * w, dtype=self._out_dtype())
        for m in modules:
            m.set_comm_manager(cm)
        self._decode_strip(z)
        cm.create_buffer()
        self.comm_manager = cm

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """`generator` is accepted and unused, as by diffusers' AutoencoderKL.decode (diffusers 0.24's pipelines pass it)."""
        cfg = self.view
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        if z.dtype != torch.float16 or not z.is_cuda:
            raise RuntimeError(f"DistriAutoencoderKLPP decodes fp16 CUDA latents only (got {z.dtype} on {z.device})")
        b, _, h, w = z.shape
        units = vae_row_plan(h, n)
        key = (tuple(z.shape), self.upcast, self._out_dtype())
        if key != self._layout_key:
            self._lay_out(z)
            self._layout_key = key
        cm = self.comm_manager
        if cm is not None:
            cm.step_begin(0)
        strip = self._decode_strip(z)
        if cm is not None:
            C, H, W = strip.shape[1], 8 * h, 8 * w
            if self.output_buffer is None:
                self.output_buffer = torch.empty((b, C, H, W), device=z.device, dtype=strip.dtype)
            strip = strip.contiguous()
            hs = strip.shape[2]
            assert tuple(strip.shape) == (b, C, 8 * units[r], W) and strip.dtype == self.output_buffer.dtype
            _lib.check(_lib.lib().df_output_gather_2d_dtype(cm.world, strip.data_ptr(), self.output_buffer.data_ptr(), b, C, H,
                                                            W, b, hs, W, 0, 8 * row_offset(units, r), 0, 0, cm.output_off,
                                                            _lib.dtype_code(strip.dtype), torch.cuda.current_stream().cuda_stream),
                       "df_output_gather_2d_dtype")
            cm.join()
            image = self.output_buffer.clone()
        else:
            image = strip.contiguous()
        for m in self._modules_pp():
            m.set_counter(0)
        return DecoderOutput(image) if return_dict else (image,)

    def close(self):
        if self.comm_manager is not None:
            self.comm_manager.close()
