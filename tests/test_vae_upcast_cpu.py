"""CPU checks of the upcast VAE decode (DistriAutoencoderKLPP(upcast=True)): diffusers' precision split on the modules, the
config the pipelines see, the refusals that stay, the compat decoder's cast after the mid block, and diffusers 0.24's SDXL
needs_upcasting branch through the fake diffusers (tests/run_from_pretrained_vae_upcast.py)."""
import os
import subprocess
import sys

import pytest
import torch
from torch.nn import functional as F

from distrifuser_b200.compat.vae import SD15_VAE, SDXL_VAE, AutoencoderKL
from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
from distrifuser_b200.modules.base_module import BaseModule
from distrifuser_b200.utils import DistriConfig

TINY = dict(SD15_VAE, block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=8)


def _dtypes(module):
    return {p.dtype for p in module.parameters()}


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_upcast_applies_diffusers_split(dtype):
    vae = AutoencoderKL(**SDXL_VAE).to(dtype)
    pp = DistriAutoencoderKLPP(vae, DistriConfig(height=64, width=64), upcast=True)
    dec = vae.decoder
    for m in (vae.post_quant_conv, dec.conv_in, dec.mid_block):
        assert _dtypes(m) == {torch.float16}
    for m in (dec.up_blocks, dec.conv_norm_out, dec.conv_out):
        assert _dtypes(m) == {torch.float32}
    assert pp.dtype == torch.float16
    # the wrappers of the fp32 part take fp32; the mid block's keep refusing it
    for part, allowed in ((dec.up_blocks, True), (dec.conv_norm_out, True), (dec.conv_out, True), (dec.mid_block, False),
                          (dec.conv_in, False)):
        wrappers = [m for m in part.modules() if isinstance(m, BaseModule)]
        assert wrappers and all(m.allow_fp32 == allowed for m in wrappers)


def test_upcast_config_is_a_copy():
    vae = AutoencoderKL(**SDXL_VAE)
    before = dict(vae.config)
    pp = DistriAutoencoderKLPP(vae, DistriConfig(height=64, width=64), upcast=True)
    assert pp.config.force_upcast is False and pp.config["force_upcast"] is False
    assert dict(vae.config) == before and vae.config.force_upcast is True
    assert {k: v for k, v in pp.config.items() if k != "force_upcast"} == {k: v for k, v in before.items() if k != "force_upcast"}
    assert pp.config.scaling_factor == SDXL_VAE["scaling_factor"]


def test_without_upcast_the_refusal_stays():
    with pytest.raises(ValueError, match="force_upcast") as e:
        DistriAutoencoderKLPP(AutoencoderKL(**SDXL_VAE), DistriConfig(height=64, width=64))
    assert "upcast=True" in str(e.value)
    pp = DistriAutoencoderKLPP(AutoencoderKL(**SD15_VAE), DistriConfig(height=64, width=64))   # fp16-safe VAE: as before
    assert not pp.upcast and pp.config is pp.vae.config
    assert not any(m.allow_fp32 for m in pp.vae.decoder.modules() if isinstance(m, BaseModule))


def test_unet_wrappers_refuse_fp32():
    from distrifuser_b200.modules.pp.groupnorm import DistriGroupNorm
    gn = DistriGroupNorm(torch.nn.GroupNorm(8, 32), DistriConfig(height=64, width=64))
    with pytest.raises(RuntimeError, match="runs fp16 tensors on a CUDA device only"):
        gn(torch.zeros(1, 32, 4, 4))


def test_vae_upcast_needs_a_distributed_vae():
    from distrifuser_b200.pipelines import DistriSDXLPipeline
    with pytest.raises(ValueError, match="pass vae="):
        DistriSDXLPipeline.from_synthetic(DistriConfig(height=64, width=64), vae_upcast=True)


def _diffusers_decoder_forward(dec, z):
    """diffusers 0.24 Decoder.forward (no gradient checkpointing): the mid block's output goes to the up blocks' dtype."""
    upscale_dtype = next(iter(dec.up_blocks.parameters())).dtype
    x = dec.conv_in(z)
    x = dec.mid_block(x).to(upscale_dtype)
    for blk in dec.up_blocks:
        x = blk(x)
    x = dec.conv_act(dec.conv_norm_out(x))
    return dec.conv_out(x)


def test_compat_decoder_casts_like_diffusers():
    """The split with fp32 standing in for fp16 and fp64 for fp32 (CPU): the compat decoder is diffusers' cast order."""
    torch.manual_seed(4)
    vae = AutoencoderKL(**TINY).eval()
    for p in vae.parameters():
        p.data.normal_(0, 0.2)
    z = torch.randn(1, 4, 5, 6)
    with torch.no_grad():
        same = vae.decode(z).sample
        for part in ("up_blocks", "conv_norm_out", "conv_out"):
            getattr(vae.decoder, part).double()
        got = vae.decode(z).sample
        want = _diffusers_decoder_forward(vae.decoder, vae.post_quant_conv(z))
    assert got.dtype == torch.float64 and torch.equal(got, want)
    assert (got - same.double()).abs().max().item() < 1e-4         # the same decode, in more precision


def test_compat_decoder_cast_is_a_noop_at_one_dtype():
    torch.manual_seed(5)
    vae = AutoencoderKL(**TINY).eval()
    z = torch.randn(1, 4, 3, 4)
    with torch.no_grad():
        dec = vae.decoder
        want = dec.conv_out(F.silu(dec.conv_norm_out(dec.up_blocks[3](dec.up_blocks[2](dec.up_blocks[1](dec.up_blocks[0](
            dec.mid_block(dec.conv_in(vae.post_quant_conv(z))))))))))
        assert torch.equal(vae.decode(z).sample, want)


def test_fake_diffusers_sdxl_needs_upcasting_branch():
    """diffusers 0.24 SDXL's needs_upcasting is False on the wrapper; the refusals of vae_upcast without distributed_vae."""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "run_from_pretrained_vae_upcast.py"), "cpu"], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "OK from_pretrained vae_upcast cpu" in r.stdout, r.stdout + r.stderr
