"""CPU checks of the patch-parallel VAE decode: the compat decoder's diffusers names and parameter count, an fp32 restatement of
the split decode (strips, halo rows after each upsampler, row-weighted GroupNorm statistics, K/V segments) against the
one-device decode, the row plan, and the public checks (force_upcast, output_type)."""
import copy
from types import SimpleNamespace

import pytest
import torch
from torch.nn import functional as F

from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline
from distrifuser_b200.compat.vae import SD15_VAE, SDXL_VAE, AutoencoderKL
from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP, vae_row_plan
from distrifuser_b200.utils import DistriConfig, split_units

TINY = dict(SD15_VAE, block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=8)


def _expected_params(cfg):
    """Parameter count of the decoder half from the config alone (diffusers 0.24 layer list)."""
    boc, G, lat = list(cfg["block_out_channels"]), cfg["norm_num_groups"], cfg["latent_channels"]
    conv = lambda ci, co, k: ci * co * k * k + co
    gn = lambda c: 2 * c
    res = lambda ci, co: gn(ci) + conv(ci, co, 3) + gn(co) + conv(co, co, 3) + (conv(ci, co, 1) if ci != co else 0)
    top = boc[-1]
    n = conv(lat, lat, 1) + conv(lat, top, 3)
    n += 2 * res(top, top) + gn(top) + 4 * (top * top + top)                      # mid block: 2 resnets + attention
    rev, out_c = list(reversed(boc)), top
    for i, c in enumerate(rev):
        prev, out_c = out_c, c
        n += res(prev, c) + cfg["layers_per_block"] * res(c, c)
        if i < len(rev) - 1:
            n += conv(c, c, 3)
    return n + gn(boc[0]) + conv(boc[0], cfg["out_channels"], 3)


@pytest.mark.parametrize("cfg", [SD15_VAE, SDXL_VAE, TINY], ids=["sd15", "sdxl", "tiny"])
def test_compat_decoder_names_and_count(cfg):
    with torch.device("meta"):
        vae = AutoencoderKL(**cfg)
    keys = set(vae.state_dict())
    assert sum(p.numel() for p in vae.parameters()) == _expected_params(cfg)
    top = cfg["block_out_channels"][-1]
    for k in ["post_quant_conv.weight", "post_quant_conv.bias", "decoder.conv_in.weight", "decoder.conv_norm_out.weight",
              "decoder.conv_out.bias", "decoder.mid_block.resnets.0.norm1.weight", "decoder.mid_block.resnets.1.conv2.weight",
              "decoder.mid_block.attentions.0.group_norm.weight", "decoder.mid_block.attentions.0.to_q.bias",
              "decoder.mid_block.attentions.0.to_k.weight", "decoder.mid_block.attentions.0.to_v.bias",
              "decoder.mid_block.attentions.0.to_out.0.weight", "decoder.up_blocks.0.upsamplers.0.conv.weight",
              "decoder.up_blocks.3.resnets.0.conv_shortcut.weight", "decoder.up_blocks.3.resnets.0.norm1.bias"]:
        assert k in keys, k
    assert not any("upsamplers" in k for k in keys if k.startswith("decoder.up_blocks.3."))     # the last block does not upsample
    assert not any(k.startswith(("encoder.", "quant_conv.")) for k in keys)
    assert vae.decoder.mid_block.attentions[0].to_q.weight.shape == (top, top)
    # layers_per_block + 1 resnets per up block, 8 tensors each (norm1, conv1, norm2, conv2; 512 -> 512: no shortcut)
    assert sum(1 for k in keys if k.startswith("decoder.up_blocks.0.resnets.")) == 8 * (cfg["layers_per_block"] + 1)


# ---------------------------------------------------------------------------------------------------- split-decode restatement
def _gn_split(norm, strips, silu):
    """GroupNorm of the whole image from per-strip moments weighted by rows (biased variance, as nn.GroupNorm)."""
    G, eps = norm.num_groups, norm.eps
    rows = [s.shape[2] for s in strips]
    mom = []
    for s in strips:
        b, c, h, w = s.shape
        g = s.reshape(b, G, -1)
        mom.append((g.mean(-1), (g * g).mean(-1)))
    mean = sum(m[0] * r for m, r in zip(mom, rows)) / sum(rows)
    meansq = sum(m[1] * r for m, r in zip(mom, rows)) / sum(rows)
    inv = (meansq - mean * mean + eps).rsqrt()
    out = []
    for s in strips:
        b, c, h, w = s.shape
        y = ((s.reshape(b, G, -1) - mean[..., None]) * inv[..., None]).reshape(b, c, h, w)
        y = y * norm.weight.view(1, -1, 1, 1) + norm.bias.view(1, -1, 1, 1)
        out.append(F.silu(y) if silu else y)
    return out


def _conv_halo(conv, strips):
    """3x3 conv of each strip with its neighbours' boundary rows (zero rows at the image border)."""
    out = []
    for r, s in enumerate(strips):
        top = strips[r - 1][:, :, -1:] if r > 0 else torch.zeros_like(s[:, :, :1])
        bot = strips[r + 1][:, :, :1] if r + 1 < len(strips) else torch.zeros_like(s[:, :, :1])
        out.append(F.conv2d(torch.cat([top, s, bot], 2), conv.weight, conv.bias, padding=(0, 1)))
    return out


def _resnet(blk, strips):
    h = _conv_halo(blk.conv1, _gn_split(blk.norm1, strips, True))
    h = _conv_halo(blk.conv2, _gn_split(blk.norm2, h, True))
    x = [blk.conv_shortcut(s) for s in strips] if blk.conv_shortcut is not None else strips
    return [a + b for a, b in zip(x, h)]


def _attention(attn, strips):
    """Each strip's queries against the K/V segments of every strip, walked from its own segment on."""
    n = len(strips)
    toks = [t.flatten(2).transpose(1, 2) for t in _gn_split(attn.group_norm, strips, False)]
    kv = [(attn.to_k(t), attn.to_v(t)) for t in toks]
    out = []
    for r, (s, t) in enumerate(zip(strips, toks)):
        order = [(r + o) % n for o in range(n)]
        k = torch.cat([kv[i][0] for i in order], 1)
        v = torch.cat([kv[i][1] for i in order], 1)
        o = F.scaled_dot_product_attention(attn.to_q(t)[:, None], k[:, None], v[:, None])[:, 0]
        o = attn.to_out[0](o).transpose(1, 2).reshape(s.shape)
        out.append(o + s)
    return out


def split_decode(vae, z, n):
    """The patch-parallel decode of rank strips of split_units(latent rows, n), one rank after the other, in fp32."""
    dec = vae.decoder
    z = vae.post_quant_conv(z)
    units = split_units(z.shape[2], n)
    zp = F.pad(z, (0, 0, 1, 1))
    strips, r0 = [], 0
    for u in units:                                                  # conv_in: each rank's rows of the whole latent
        strips.append(F.conv2d(zp[:, :, r0:r0 + u + 2], dec.conv_in.weight, dec.conv_in.bias, padding=(0, 1)))
        r0 += u
    mid = dec.mid_block
    strips = _resnet(mid.resnets[0], strips)
    strips = _resnet(mid.resnets[1], _attention(mid.attentions[0], strips))
    for blk in dec.up_blocks:
        for res in blk.resnets:
            strips = _resnet(res, strips)
        if blk.upsamplers is not None:
            strips = _conv_halo(blk.upsamplers[0].conv, [F.interpolate(s, scale_factor=2.0, mode="nearest") for s in strips])
    strips = _conv_halo(dec.conv_out, _gn_split(dec.conv_norm_out, strips, True))
    assert [s.shape[2] for s in strips] == [8 * u for u in units]
    return torch.cat(strips, 2)


@pytest.mark.parametrize("n,rows,cols", [(2, 6, 5), (3, 9, 4), (8, 10, 3)], ids=["n2", "n3-uneven-9-rows", "n8-uneven"])
def test_split_decode_equals_one_device(n, rows, cols):
    torch.manual_seed(n)
    vae = AutoencoderKL(**TINY).eval()
    for p in vae.parameters():                                       # weights of real magnitude everywhere (biases too)
        p.data.normal_(0, 0.2)
    z = torch.randn(1, 4, rows, cols)
    with torch.no_grad():
        want = vae.decode(z).sample
        got = split_decode(vae, z, n)
    assert got.shape == want.shape == (1, 3, 8 * rows, 8 * cols)
    err = (got - want).abs().max().item()
    assert err < 1e-5 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize("world", range(1, 9))
def test_row_plan(world):
    for h in (world, world + 1, 9, 64, 128, 480):
        if h < world:
            continue
        units = vae_row_plan(h, world)
        assert len(units) == world and sum(units) == h and max(units) - min(units) <= 1 and min(units) >= 1
        assert units == sorted(units, reverse=True)                  # the first h % world ranks take the extra row
    with pytest.raises(ValueError, match="at least one latent row per rank"):
        vae_row_plan(world - 1, world)


def test_force_upcast_is_refused():
    cfg = DistriConfig(height=64, width=64)
    with pytest.raises(ValueError, match="force_upcast"):
        DistriAutoencoderKLPP(AutoencoderKL(**dict(TINY, force_upcast=True)), cfg)
    assert SDXL_VAE["force_upcast"] and not SD15_VAE["force_upcast"]


class _UNet:
    def __init__(self):
        self.config = SimpleNamespace(in_channels=4, cross_attention_dim=16)

    def __call__(self, x, t, encoder_hidden_states=None, added_cond_kwargs=None, return_dict=False):
        return (0.1 * x + 0.01 * float(t) * torch.ones_like(x),)


def test_output_type_latent_unchanged_with_vae():
    vae = AutoencoderKL(**TINY).eval()
    run = lambda pipe, **kw: pipe(prompt="x", height=32, width=48, num_inference_steps=3, guidance_scale=5.0,
                                  generator=torch.Generator().manual_seed(0), **kw).images
    plain = SyntheticLatentPipeline(_UNet(), sdxl=False, device="cpu", dtype=torch.float32)
    with_vae = SyntheticLatentPipeline(_UNet(), sdxl=False, device="cpu", dtype=torch.float32, vae=vae)
    lat = run(plain)
    assert torch.equal(run(with_vae), lat) and torch.equal(run(with_vae, output_type="latent"), lat)
    img = run(with_vae, output_type="pt")
    with torch.no_grad():
        want = (vae.decode(lat / TINY["scaling_factor"]).sample / 2 + 0.5).clamp(0, 1)
    assert img.shape == (1, 3, 32, 48) and torch.equal(img, want)
    with pytest.raises(ValueError, match="needs a VAE"):
        run(plain, output_type="pt")


def test_wrapper_leaves_the_unet_config_alone():
    """The decoder's wrappers see a world-wide, synchronous, un-split view; the caller's config is not changed."""
    cfg = DistriConfig(height=64, width=64, mode="corrected_async_gn")
    before = copy.copy(cfg.__dict__)
    pp = DistriAutoencoderKLPP(AutoencoderKL(**SD15_VAE), cfg)
    assert cfg.__dict__ == before
    assert pp.view.mode == "full_sync" and pp.view.n_device_per_batch == cfg.world_size and pp.view.split_idx() == cfg.rank
    assert pp.config.scaling_factor == SD15_VAE["scaling_factor"]


def test_decode_takes_diffusers_generator_argument():
    """diffusers 0.24's pipelines call vae.decode(latents, return_dict=False, generator=generator)."""
    pp = DistriAutoencoderKLPP(AutoencoderKL(**SD15_VAE), DistriConfig(height=64, width=64))
    with pytest.raises(RuntimeError, match="fp16 CUDA latents"):     # past the signature: a CPU latent is refused next
        pp.decode(torch.zeros(1, 4, 8, 8), return_dict=False, generator=torch.Generator())
    out = AutoencoderKL(**TINY).decode(torch.zeros(1, 4, 2, 2), return_dict=False, generator=torch.Generator())[0]
    assert out.shape == (1, 3, 16, 16)


def test_attention_width_other_than_512_is_refused():
    with pytest.raises(ValueError, match="one head of width 512"):
        DistriAutoencoderKLPP(AutoencoderKL(**TINY), DistriConfig(height=64, width=64))


def test_from_pretrained_distributed_vae_refusals():
    """from_pretrained(distributed_vae=True) through the fake diffusers: a pipeline without a VAE, and a VAE with
    force_upcast=True, raise ValueError (tests/run_from_pretrained_vae.py; the GPU modes run the decode)."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "run_from_pretrained_vae.py"), "refusals"], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "OK refusals" in r.stdout, r.stdout + r.stderr
