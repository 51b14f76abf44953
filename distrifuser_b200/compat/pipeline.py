"""A latent-space stand-in for StableDiffusion(XL)Pipeline when diffusers / checkpoints are unavailable.

It reproduces the part of the diffusers denoising loop the reference's hot path lives in (SURVEY 3.2): CFG batch
duplication, scheduler.scale_model_input, one UNet call per step, guidance combine, scheduler.step.  Prompt
encoding is replaced by seeded synthetic embeddings; with a VAE (compat.vae) output_type="pt" decodes the latents."""
import hashlib
from types import SimpleNamespace

import torch

from .schedulers import DDIMScheduler, EulerDiscreteScheduler


class SyntheticLatentPipeline:
    def __init__(self, unet, scheduler=None, sdxl: bool = True, device="cuda", dtype=torch.float16, vae=None):
        self.unet = unet
        self.vae = vae
        self.scheduler = scheduler or (EulerDiscreteScheduler() if sdxl else DDIMScheduler())
        self.sdxl = sdxl
        self.device = torch.device(device)
        self.dtype = dtype
        self.vae_scale_factor = 8
        self.text_encoder_2 = None
        self._progress = {}

    def to(self, device):
        self.device = torch.device(device)
        return self

    def set_progress_bar_config(self, **kwargs):
        self._progress = kwargs

    # -- the three helpers the reference's prepare() calls (pipelines.py:79-112,223-243)
    def encode_prompt(self, prompt="", *args, device=None, **kwargs):
        cfg = self.unet.config
        seed = int.from_bytes(hashlib.sha256(str(prompt).encode()).digest()[:4], "little")
        g = torch.Generator().manual_seed(seed)
        embeds = torch.randn(1, 77, cfg.cross_attention_dim, generator=g).to(self.device, self.dtype)
        if not self.sdxl:
            return embeds, None
        pooled_dim = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
        pooled = torch.randn(1, pooled_dim, generator=g).to(self.device, self.dtype)
        return embeds, None, pooled, None

    def prepare_latents(self, batch_size, num_channels, height, width, dtype, device, generator, latents=None):
        shape = (batch_size, num_channels, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if latents is None:
            gdev = generator.device if generator is not None else torch.device("cpu")
            latents = torch.randn(shape, generator=generator, device=gdev, dtype=torch.float32)
        return latents.to(device=device, dtype=dtype) * self.scheduler.init_noise_sigma

    def _get_add_time_ids(self, original_size, crops_coords_top_left, target_size, dtype, text_encoder_projection_dim=None):
        return torch.tensor([list(original_size + crops_coords_top_left + target_size)], dtype=dtype)

    @torch.no_grad()
    def __call__(self, prompt="", height=1024, width=1024, num_inference_steps=50, guidance_scale=5.0, generator=None,
                 latents=None, output_type="latent", prompt_embeds=None, pooled_prompt_embeds=None, image=None,
                 controlnet_conditioning_scale=1.0, **kwargs):
        """image: the ControlNet conditioning image [1, 3, height, width] when the UNet has a ControlNet attached.
        output_type: "pt" returns the VAE's image in [0, 1], [1, 3, height, width] (needs a VAE); anything else the final latents."""
        if output_type == "pt" and self.vae is None:
            raise ValueError("output_type='pt' needs a VAE: build the pipeline with vae=AutoencoderKL(...)")
        dev = self.device
        cfg_on = guidance_scale > 1.0
        if prompt_embeds is None:
            enc = self.encode_prompt(prompt)
            prompt_embeds, pooled_prompt_embeds = enc[0], (enc[2] if self.sdxl else None)
            neg = self.encode_prompt("")
            neg_embeds, neg_pooled = neg[0], (neg[2] if self.sdxl else None)
        else:  # host tensors supplied by the caller: [uncond | cond] stacked on dim 0 when CFG is on
            prompt_embeds = prompt_embeds.to(dev, self.dtype, non_blocking=True)
            if pooled_prompt_embeds is not None:
                pooled_prompt_embeds = pooled_prompt_embeds.to(dev, self.dtype, non_blocking=True)
            neg_embeds = neg_pooled = None
        if cfg_on and neg_embeds is not None:
            prompt_embeds = torch.cat([neg_embeds, prompt_embeds], 0)
            if self.sdxl:
                pooled_prompt_embeds = torch.cat([neg_pooled, pooled_prompt_embeds], 0)
        B = prompt_embeds.shape[0]
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        lat = self.prepare_latents(1, self.unet.config.in_channels, height, width, torch.float32, dev, generator, latents)
        added = None
        if self.sdxl:
            ids = self._get_add_time_ids((height, width), (0, 0), (height, width), self.dtype).to(dev).repeat(B, 1)
            added = {"text_embeds": pooled_prompt_embeds, "time_ids": ids}
        control = {}
        if image is not None:                                        # both CFG branches get the same conditioning image
            cond = image.to(dev, self.dtype)
            control = dict(controlnet_cond=torch.cat([cond] * 2) if cfg_on else cond,
                           conditioning_scale=controlnet_conditioning_scale)
        for i in range(num_inference_steps):
            t = self.scheduler.timesteps[i]
            x = torch.cat([lat] * 2) if cfg_on else lat
            x = self.scheduler.scale_model_input(x, t).to(self.dtype)
            eps = self.unet(x, t, encoder_hidden_states=prompt_embeds, added_cond_kwargs=added, return_dict=False,
                            **control)[0]
            if cfg_on:
                e_u, e_c = eps.float().chunk(2)
                eps = e_u + guidance_scale * (e_c - e_u)
            lat = self.scheduler.step(eps, t, lat)[0]
        if output_type == "pt":                                      # diffusers: decode, then the image processor's denormalise
            image = self.vae.decode((lat / self.vae.config.scaling_factor).to(self.dtype), return_dict=False,
                                    generator=generator)[0]
            return SimpleNamespace(images=(image / 2 + 0.5).clamp(0, 1))
        return SimpleNamespace(images=lat)
