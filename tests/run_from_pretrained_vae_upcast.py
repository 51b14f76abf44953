"""TEST INFRASTRUCTURE -- DistriSDXLPipeline.from_pretrained(cfg, distributed_vae=True, vae_upcast=True) with the stock SDXL VAE
config (force_upcast=True) in a fresh interpreter, on the fake diffusers of run_from_pretrained_vae.py, whose pipeline here
ends every call as diffusers 0.24's StableDiffusionXLPipeline does with a VAE:
    needs_upcasting = self.vae.dtype == torch.float16 and self.vae.config.force_upcast
    if needs_upcasting:
        self.upcast_vae()
        latents = latents.to(next(iter(self.vae.post_quant_conv.parameters())).dtype)
    image = self.vae.decode(latents / self.vae.config.scaling_factor, return_dict=False)[0]
    if needs_upcasting:
        self.vae.to(dtype=torch.float16)
The wrapper reports force_upcast=False and dtype fp16, so upcast_vae() -- which would move the wrapper to fp32 and look up
the mid-block attention's processor, which the wrapper does not have -- must never run, and decode() must get fp16 latents.
    python tests/run_from_pretrained_vae_upcast.py cpu     # the refusals, and the wrapper as the pipeline sees it
    python tests/run_from_pretrained_vae_upcast.py gpu     # the whole pipeline call, image = fp32 decode of its latents"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import run_from_pretrained_vae as base  # noqa: E402  (installs the fake diffusers and its 0.24 decode)
import torch  # noqa: E402

from run_from_pretrained import TINY_SDXL  # noqa: E402
from distrifuser_b200.compat.vae import SDXL_VAE  # noqa: E402

UPCAST_CALLS = []
DECODE_DTYPES = []


class PipelineSDXL024(base.Pipeline024):
    """Pipeline024 with the needs_upcasting branch of diffusers 0.24's StableDiffusionXLPipeline.__call__."""

    def upcast_vae(self):                                            # diffusers 0.24, torch 2 attention processors
        UPCAST_CALLS.append(type(self.vae).__name__)
        dtype = self.vae.dtype
        self.vae.to(dtype=torch.float32)
        self.vae.decoder.mid_block.attentions[0].processor      # noqa: B018  (diffusers reads it here)
        self.vae.post_quant_conv.to(dtype)
        self.vae.decoder.conv_in.to(dtype)
        self.vae.decoder.mid_block.to(dtype)

    def __call__(self, *args, output_type="pil", generator=None, **kwargs):
        latents = super(base.Pipeline024, self).__call__(*args, output_type="latent", generator=generator, **kwargs).images
        if output_type == "latent":
            return type("Out", (), {"images": latents})()
        latents = latents.to(self.vae.dtype)                         # the UNet's dtype in diffusers
        needs_upcasting = self.vae.dtype == torch.float16 and self.vae.config.force_upcast
        if needs_upcasting:
            self.upcast_vae()
            latents = latents.to(next(iter(self.vae.post_quant_conv.parameters())).dtype)
        DECODE_DTYPES.append(latents.dtype)
        image = self.vae.decode(latents / self.vae.config.scaling_factor, return_dict=False)[0]
        if needs_upcasting:
            self.vae.to(dtype=torch.float16)
        return type("Out", (), {"images": (image / 2 + 0.5).clamp(0, 1)})()


def _sdxl_from_pretrained(original):
    def from_pretrained(cls, *args, **kw):
        pipe = original.__func__(cls, *args, **kw)
        pipe.__class__ = PipelineSDXL024
        return pipe
    return classmethod(from_pretrained)


base.diffusers._Pipeline.from_pretrained = _sdxl_from_pretrained(base.diffusers._Pipeline.from_pretrained)


def _pipe(**kw):
    from distrifuser_b200.pipelines import DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    base.diffusers.UNET_CONFIG.clear()
    base.diffusers.UNET_CONFIG.update(TINY_SDXL)
    base.VAE_CONFIG["config"] = SDXL_VAE
    cfg = DistriConfig(height=256, width=256, warmup_steps=1)
    return DistriSDXLPipeline.from_pretrained(cfg, pretrained_model_name_or_path="fake/checkpoint", **kw)


def _check_wrapper(vae):
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    assert isinstance(vae, DistriAutoencoderKLPP) and vae.upcast
    assert vae.dtype == torch.float16 and vae.config.force_upcast is False
    assert not (vae.dtype == torch.float16 and vae.config.force_upcast)   # needs_upcasting
    assert vae.vae.config.force_upcast is True                      # the caller's VAE config is not mutated
    assert vae.vae.decoder.up_blocks[0].resnets[0].conv1.module.weight.dtype == torch.float32


def main():
    what = sys.argv[1]
    if what == "cpu":                                                # the pipeline's prepare() runs the UNet: GPU only
        base._raises(lambda: _pipe(vae_upcast=True), "distributed_vae=True")
        base._raises(lambda: _pipe(distributed_vae=False, vae_upcast=True), "distributed_vae=True")
        base._raises(lambda: _pipe(distributed_vae=True), "force_upcast")          # without vae_upcast: refused as before
        from distrifuser_b200.compat.vae import AutoencoderKL
        from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
        from distrifuser_b200.utils import DistriConfig
        _check_wrapper(DistriAutoencoderKLPP(AutoencoderKL(**SDXL_VAE).half(), DistriConfig(height=256, width=256), upcast=True))
        print("OK from_pretrained vae_upcast cpu")
        return
    pipe = _pipe(distributed_vae=True, vae_upcast=True)
    vae = pipe.pipeline.vae
    _check_wrapper(vae)
    run = lambda **kw: pipe(prompt="a photo", num_inference_steps=3, guidance_scale=5.0,
                            generator=torch.Generator().manual_seed(0), **kw).images
    image = run()
    assert UPCAST_CALLS == [], UPCAST_CALLS
    assert DECODE_DTYPES == [torch.float16], DECODE_DTYPES
    assert image.dtype == torch.float32 and image.shape == (1, 3, 256, 256) and torch.isfinite(image).all()
    lat = run(output_type="latent")
    want = vae.decode(lat.half() / SDXL_VAE["scaling_factor"], return_dict=False)[0]
    assert want.dtype == torch.float32
    assert torch.equal(image, (want / 2 + 0.5).clamp(0, 1))
    print("OK from_pretrained vae_upcast gpu")


if __name__ == "__main__":
    main()
