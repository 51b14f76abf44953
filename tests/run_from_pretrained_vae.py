"""TEST INFRASTRUCTURE -- drives Distri{SDXL,SD}Pipeline.from_pretrained(cfg, distributed_vae=True) in a fresh interpreter whose
`diffusers` is tests/fake_diffusers, extended here with what diffusers 0.24's StableDiffusion(XL)Pipeline does with its VAE:
the pipeline carries `vae`, and every call whose output_type is not "latent" ("pil" by default) ends with
    image = self.vae.decode(latents / self.vae.config.scaling_factor, return_dict=False, generator=generator)[0]
and the image processor's denormalisation (image / 2 + 0.5).clamp(0, 1).
    python tests/run_from_pretrained_vae.py refusals     # CPU: no VAE, and a force_upcast VAE, raise ValueError
    python tests/run_from_pretrained_vae.py sd15|sdxl    # GPU: from_pretrained(distributed_vae=True) -> prepare() -> __call__
What this fake cannot show: diffusers' own ResnetBlock2D / Upsample2D / Attention / Decoder classes under the wrappers (the
compat restatement stands in for them), and DiffusionPipeline.__setattr__ re-registering `vae` in the pipeline config."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "fake_diffusers"))

import diffusers  # noqa: E402  (the fake)
import torch  # noqa: E402

from run_from_pretrained import TINY_SD15, TINY_SDXL  # noqa: E402
from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline  # noqa: E402
from distrifuser_b200.compat.vae import SD15_VAE, SDXL_VAE, AutoencoderKL  # noqa: E402

VAE_CONFIG = {}           # the VAE the fake pipelines load (None: a pipeline without one)
DECODE_CALLS = []


class Pipeline024(SyntheticLatentPipeline):
    """The latent pipeline plus diffusers 0.24's decode at the end of __call__."""

    def to(self, device):                                            # DiffusionPipeline.to moves every module
        if self.vae is not None:
            self.vae.to(device)
        return super().to(device)

    def __call__(self, *args, output_type="pil", generator=None, **kwargs):
        latents = super().__call__(*args, output_type="latent", generator=generator, **kwargs).images
        if output_type == "latent":
            return type("Out", (), {"images": latents})()
        DECODE_CALLS.append(type(self.vae).__name__)
        image = self.vae.decode(latents.to(self.vae.dtype) / self.vae.config.scaling_factor, return_dict=False,
                                generator=generator)[0]
        return type("Out", (), {"images": (image / 2 + 0.5).clamp(0, 1)})()


def _from_pretrained(original):
    def from_pretrained(cls, name, torch_dtype=torch.float32, unet=None, **kw):
        pipe = original.__func__(cls, name, torch_dtype=torch_dtype, unet=unet, **kw)    # the fake's own type checks
        vae = None
        if VAE_CONFIG.get("config") is not None:
            torch.manual_seed(0)
            vae = AutoencoderKL(**VAE_CONFIG["config"]).to(torch_dtype).eval()
        return Pipeline024(pipe.unet, None, sdxl=cls.sdxl, device="cpu", dtype=torch_dtype, vae=vae)
    return classmethod(from_pretrained)


diffusers._Pipeline.from_pretrained = _from_pretrained(diffusers._Pipeline.from_pretrained)


def _pipe(what, vae_config, distributed_vae=True):
    """distributed_vae=None: the argument is not passed."""
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    sdxl = what == "sdxl"
    diffusers.UNET_CONFIG.clear()
    diffusers.UNET_CONFIG.update(TINY_SDXL if sdxl else TINY_SD15)
    VAE_CONFIG["config"] = vae_config
    cfg = DistriConfig(height=256, width=256, warmup_steps=1)
    cls = DistriSDXLPipeline if sdxl else DistriSDPipeline
    kw = {} if distributed_vae is None else dict(distributed_vae=distributed_vae)
    return cls.from_pretrained(cfg, pretrained_model_name_or_path="fake/checkpoint", **kw)


def _raises(fn, match):
    try:
        fn()
    except ValueError as e:
        assert match in str(e), e
        return
    raise AssertionError(f"no ValueError ({match})")


def main():
    what = sys.argv[1]
    if what == "refusals":
        _raises(lambda: _pipe("sd15", None), "has no VAE")
        _raises(lambda: _pipe("sdxl", SDXL_VAE), "force_upcast")
        print("OK refusals")
        return
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    vae_config = SD15_VAE if what == "sd15" else dict(SDXL_VAE, force_upcast=False)      # SDXL: an fp16-fixed VAE
    pipe = _pipe(what, vae_config)
    assert isinstance(pipe.pipeline.vae, DistriAutoencoderKLPP)
    run = lambda **kw: pipe(prompt="a photo", num_inference_steps=3, guidance_scale=5.0,
                            generator=torch.Generator().manual_seed(0), **kw).images
    image = run()                                                    # output_type "pil": the decode passes generator=
    assert DECODE_CALLS == ["DistriAutoencoderKLPP"], DECODE_CALLS
    assert image.shape == (1, 3, 256, 256) and image.min() >= 0 and image.max() <= 1 and torch.isfinite(image).all()
    lat = run(output_type="latent")
    want = pipe.pipeline.vae.decode(lat.half() / vae_config["scaling_factor"], return_dict=False)[0]
    assert torch.equal(image, (want / 2 + 0.5).clamp(0, 1))
    plain = _pipe(what, vae_config, distributed_vae=None)            # off by default: the pipeline's VAE is left alone
    assert isinstance(plain.pipeline.vae, AutoencoderKL)
    print("OK from_pretrained distributed_vae", what)


if __name__ == "__main__":
    main()
