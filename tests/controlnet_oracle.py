"""TEST INFRASTRUCTURE -- fp32 oracle of UNet + ControlNet, and the drivers of the ControlNet parity tests.

StubControlNetModel restates diffusers 0.24's ControlNetModel on the diffusers stub's blocks (oracle/diffusers_stub), with its
parameter names, so that the product's compat ControlNetModel loads its state_dict strict=True.  unet_forward() is the stub
UNet's forward with diffusers' residual inputs: skip i + residual i, and the mid-block output + the mid residual.

The patch-parallel oracle is the existing one (oracle/pp_modules.OracleUNetPP) around a module that runs both models: its
module surgery wraps the ControlNet's layers exactly like the UNet's, each model's first conv (`conv_in`, the latent one and the
conditioning network's) slices this rank's rows, and both models read one-step-stale data on the same step clock."""
from __future__ import annotations

import os
import sys

import torch
from torch import nn
from torch.nn import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from diffusers.models.unet_2d_condition import (CrossAttnDownBlock2D, DownBlock2D, TimestepEmbedding, Timesteps,  # noqa: E402
                                                UNetMidBlock2DCrossAttn, sdxl_config)


class StubControlNetConditioningEmbedding(nn.Module):
    def __init__(self, emb_channels, cond_channels=3, block_out_channels=(16, 32, 96, 256)):
        super().__init__()
        self.conv_in = nn.Conv2d(cond_channels, block_out_channels[0], kernel_size=3, padding=1)
        self.blocks = nn.ModuleList([])
        for i in range(len(block_out_channels) - 1):
            cin, cout = block_out_channels[i], block_out_channels[i + 1]
            self.blocks.append(nn.Conv2d(cin, cin, kernel_size=3, padding=1))
            self.blocks.append(nn.Conv2d(cin, cout, kernel_size=3, padding=1, stride=2))
        self.conv_out = nn.Conv2d(block_out_channels[-1], emb_channels, kernel_size=3, padding=1)
        nn.init.zeros_(self.conv_out.weight)
        nn.init.zeros_(self.conv_out.bias)

    def forward(self, conditioning):
        embedding = F.silu(self.conv_in(conditioning))
        for block in self.blocks:
            embedding = F.silu(block(embedding))
        return self.conv_out(embedding)


def _zero_conv(c):
    conv = nn.Conv2d(c, c, kernel_size=1)
    nn.init.zeros_(conv.weight)
    nn.init.zeros_(conv.bias)
    return conv


class StubControlNetModel(nn.Module):
    """diffusers 0.24 ControlNetModel for the SD1.x / SDXL configurations (controlnet.py), without the options they leave off."""

    def __init__(self, **cfg):
        super().__init__()
        full = sdxl_config()
        full.update(cfg)
        from types import SimpleNamespace
        self.config = SimpleNamespace(**full)
        c = self.config
        boc = tuple(c.block_out_channels)
        temb = boc[0] * 4
        g, eps = c.norm_num_groups, c.norm_eps
        heads, depth = tuple(c.attention_head_dim), tuple(c.transformer_layers_per_block)
        self.conv_in = nn.Conv2d(c.in_channels, boc[0], 3, padding=1)
        self.time_proj = Timesteps(boc[0], True, 0)
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        if c.addition_embed_type == "text_time":
            self.add_time_proj = Timesteps(c.addition_time_embed_dim, True, 0)
            self.add_embedding = TimestepEmbedding(c.projection_class_embeddings_input_dim, temb)
        self.controlnet_cond_embedding = StubControlNetConditioningEmbedding(boc[0])
        self.down_blocks = nn.ModuleList([])
        self.controlnet_down_blocks = nn.ModuleList([_zero_conv(boc[0])])
        out_ch = boc[0]
        for i, t in enumerate(c.down_block_types):
            in_ch, out_ch = out_ch, boc[i]
            final = i == len(boc) - 1
            cls = CrossAttnDownBlock2D if t == "CrossAttnDownBlock2D" else DownBlock2D
            self.down_blocks.append(cls(in_ch, out_ch, temb, c.layers_per_block, g, eps, not final, heads=heads[i],
                                        depth=depth[i], cross_dim=c.cross_attention_dim, linear_proj=c.use_linear_projection))
            for _ in range(c.layers_per_block):
                self.controlnet_down_blocks.append(_zero_conv(out_ch))
            if not final:
                self.controlnet_down_blocks.append(_zero_conv(out_ch))
        self.controlnet_mid_block = _zero_conv(boc[-1])
        self.mid_block = UNetMidBlock2DCrossAttn(boc[-1], temb, g, eps, heads[-1], depth[-1], c.cross_attention_dim,
                                                 c.use_linear_projection)

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                added_cond_kwargs=None):
        timesteps = timestep
        if not torch.is_tensor(timesteps):
            timesteps = torch.tensor([timesteps], dtype=torch.int64, device=sample.device)
        elif timesteps.ndim == 0:
            timesteps = timesteps[None].to(sample.device)
        timesteps = timesteps.expand(sample.shape[0])
        emb = self.time_embedding(self.time_proj(timesteps).to(sample.dtype))
        if self.config.addition_embed_type == "text_time":
            text_embeds, time_ids = added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"]
            time_embeds = self.add_time_proj(time_ids.flatten()).reshape(text_embeds.shape[0], -1)
            emb = emb + self.add_embedding(torch.cat([text_embeds, time_embeds], dim=-1).to(emb.dtype))
        sample = self.conv_in(sample)
        sample = sample + self.controlnet_cond_embedding(controlnet_cond)
        down = (sample,)
        for blk in self.down_blocks:
            sample, res = blk(sample, emb, encoder_hidden_states=encoder_hidden_states)
            down += res
        sample = self.mid_block(sample, emb, encoder_hidden_states=encoder_hidden_states)
        down = [blk(s) * conditioning_scale for s, blk in zip(down, self.controlnet_down_blocks)]
        return down, self.controlnet_mid_block(sample) * conditioning_scale


def unet_forward(unet, sample, timestep, encoder_hidden_states, added_cond_kwargs=None, down_res=None, mid_res=None):
    """The stub UNet's forward with diffusers' down_block_additional_residuals / mid_block_additional_residual."""
    timesteps = timestep
    if not torch.is_tensor(timesteps):
        timesteps = torch.tensor([timesteps], dtype=torch.int64, device=sample.device)
    elif timesteps.ndim == 0:
        timesteps = timesteps[None].to(sample.device)
    timesteps = timesteps.expand(sample.shape[0])
    emb = unet.time_embedding(unet.time_proj(timesteps).to(sample.dtype))
    if unet.config.addition_embed_type == "text_time":
        text_embeds, time_ids = added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"]
        time_embeds = unet.add_time_proj(time_ids.flatten()).reshape(text_embeds.shape[0], -1)
        emb = emb + unet.add_embedding(torch.cat([text_embeds, time_embeds], dim=-1).to(emb.dtype))
    sample = unet.conv_in(sample)
    res = (sample,)
    for blk in unet.down_blocks:
        sample, out = blk(sample, emb, encoder_hidden_states=encoder_hidden_states)
        res += out
    if down_res is not None:
        res = tuple(r + d for r, d in zip(res, down_res, strict=True))
    sample = unet.mid_block(sample, emb, encoder_hidden_states=encoder_hidden_states)
    if mid_res is not None:
        sample = sample + mid_res
    for blk in unet.up_blocks:
        n = len(blk.resnets)
        r, res = res[-n:], res[:-n]
        sample = blk(sample, r, emb, encoder_hidden_states=encoder_hidden_states)
    return unet.conv_out(unet.conv_act(unet.conv_norm_out(sample)))


def make_controlnet(family: str, seed: int = 0, zero: bool = False, dtype=torch.float32):
    """Seeded stub ControlNet.  zero=False also draws the zero-initialised layers (the conditioning network's conv_out and the
    1x1 zero convs), so that the residuals are not zero and the parity tests see them."""
    from oracle import workloads as W
    torch.manual_seed(seed + 101)
    cn = StubControlNetModel(**W.unet_config(family))
    if not zero:
        g = torch.Generator().manual_seed(seed + 202)
        with torch.no_grad():
            for conv in [cn.controlnet_cond_embedding.conv_out, *cn.controlnet_down_blocks, cn.controlnet_mid_block]:
                fan_in = conv.weight[0].numel()
                conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * (0.5 / fan_in ** 0.5))
                conv.bias.copy_(torch.randn(conv.bias.shape, generator=g) * 0.05)
    return cn.to(dtype).eval()


def cond_image(case, dtype=torch.float32):
    """Seeded conditioning image [1, 3, 8 * latent rows, 8 * latent cols] in [-1, 1] with some spatial structure."""
    S, T = case.hw
    g = torch.Generator().manual_seed(case.input_seed + 17)
    img = torch.rand(1, 3, S, T, generator=g) * 2 - 1
    return F.interpolate(img, scale_factor=8, mode="bilinear", align_corners=False).to(dtype)


class ControlledUNet(nn.Module):
    """Runs ControlNet then UNet with the UNet's call signature; the conditioning image is set per call (`cond`, batch 1, shared by
    both CFG branches).  `down_blocks` is the UNet's, so that OracleUNetPP derives the row plan from it."""

    def __init__(self, unet, controlnet, scale=1.0):
        super().__init__()
        self.unet, self.controlnet, self.scale = unet, controlnet, scale
        self.cond = None

    @property
    def down_blocks(self):
        return self.unet.down_blocks

    @property
    def config(self):
        return self.unet.config

    def forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None, return_dict=False):
        cond = self.cond.expand(sample.shape[0], -1, -1, -1)
        down, mid = self.controlnet(sample, timestep, encoder_hidden_states, cond, self.scale,
                                    added_cond_kwargs=added_cond_kwargs)
        return (unet_forward(self.unet, sample, timestep, encoder_hidden_states, added_cond_kwargs, down, mid),)


def _oracle_worker(rank, case, bessel, scale, port, outdir):
    from oracle import harness as H
    from oracle import pp_modules as P
    from oracle import workloads as W
    H._paths("oracle")
    H._init(rank, case.world_size, port)
    cfg = H._unet_config(case, rank)
    ucfg = W.unet_config(case.family)
    model = ControlledUNet(W.make_unet(case.family, case.weight_seed), make_controlnet(case.family, case.weight_seed), scale)
    model.cond = cond_image(case)
    pp = P.OracleUNetPP(model, cfg, bessel=bessel)
    outs = []
    with torch.no_grad():
        pp.prepare(W.unet_inputs(case, 0, ucfg))
        pp.set_counter(0)
        for t in range(case.steps):
            outs.append(pp(**W.unet_inputs(case, t, ucfg)).clone())
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        from torch import distributed as dist
        dist.barrier()
        dist.destroy_process_group()


def run_oracle(case, bessel=True, scale=1.0):
    """-> outs[step]: the oracle's patch-parallel UNet + ControlNet eps prediction (asserted identical on every rank)."""
    from oracle.harness import run_ranks
    per_rank = run_ranks(_oracle_worker, case, bessel, scale)
    for r in range(1, case.world_size):
        for a, b in zip(per_rank[0], per_rank[r]):
            assert torch.equal(a, b), "the output must be identical on every rank"
    return per_rank[0]


def run_one_device(case, scale=1.0):
    """-> outs[step]: plain fp32 UNet + ControlNet on one device (no wrappers)."""
    from oracle import harness as H
    from oracle import workloads as W
    H._paths("oracle")
    ucfg = W.unet_config(case.family)
    model = ControlledUNet(W.make_unet(case.family, case.weight_seed), make_controlnet(case.family, case.weight_seed), scale)
    model.cond = cond_image(case)
    with torch.no_grad():
        return [model(**W.unet_inputs(case, t, ucfg))[0] for t in range(case.steps)]


def _oracle_traj_worker(rank, case, num_steps, guidance, port, outdir):
    """Euler trajectory of the oracle UNet + ControlNet through the same latent pipeline as the product."""
    from oracle import harness as H
    from oracle import pp_modules as P
    from oracle import workloads as W
    from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline
    H._paths("oracle")
    H._init(rank, case.world_size, port)
    cfg = H._unet_config(case, rank)
    ucfg = W.unet_config(case.family)
    model = ControlledUNet(W.make_unet(case.family, case.weight_seed), make_controlnet(case.family, case.weight_seed))
    model.cond = cond_image(case)
    pp = P.OracleUNetPP(model, cfg)
    pp.prepare(W.unet_inputs(case, 0, ucfg))
    pipe = SyntheticLatentPipeline(H._OracleUNetAdapter(pp, model.config), sdxl=ucfg.get("addition_embed_type") == "text_time",
                                   device="cpu", dtype=torch.float32)
    pp.set_counter(0)
    with torch.no_grad():
        lat = pipe(prompt="a photo", height=cfg.height, width=cfg.width, num_inference_steps=num_steps,
                   guidance_scale=guidance, generator=torch.Generator().manual_seed(case.input_seed)).images
    torch.save(lat, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        from torch import distributed as dist
        dist.barrier()
        dist.destroy_process_group()


def run_oracle_trajectory(case, num_steps=8, guidance=5.0):
    from oracle.harness import run_ranks
    return run_ranks(_oracle_traj_worker, case, num_steps, guidance)[0]


# ------------------------------------------------------------------------------------------------------------ product (GPU)
def _product_init(rank, case, port):
    from torch import distributed as dist
    if case.world_size > 1:
        if torch.cuda.device_count() < case.world_size:
            os.environ["DISTRIFUSER_B200_SHARE_GPU"] = "1"
        os.environ["LOCAL_RANK"] = str(rank)
        dist.init_process_group("gloo", rank=rank, world_size=case.world_size, init_method=f"tcp://127.0.0.1:{port}")


def _product_pipe(case, use_graph, zero=False):
    """The product pipeline around the oracle's seeded weights.  zero=True: a zero-initialised ControlNet; None: no ControlNet."""
    from oracle import workloads as W
    from distrifuser_b200.compat.controlnet import ControlNetModel
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(**case.config_kwargs(), use_cuda_graph=use_graph)
    ucfg = W.unet_config(case.family)
    unet = UNet2DConditionModel(**ucfg)
    unet.load_state_dict(W.make_unet(case.family, case.weight_seed).state_dict(), strict=True)
    cn = None
    if zero is not None:
        cn = ControlNetModel(**ucfg)
        cn.load_state_dict(make_controlnet(case.family, case.weight_seed, zero=zero).state_dict(), strict=True)
    cls = DistriSDXLPipeline if ucfg.get("addition_embed_type") == "text_time" else DistriSDPipeline
    return cls.from_synthetic(cfg, unet=unet, controlnet=cn), ucfg


def _product_steps(pipe, ucfg, case, scale, with_cn):
    from oracle import workloads as W
    model, dev = pipe.pipeline.unet, pipe.distri_config.device
    cond = cond_image(case).to(dev, torch.float16).expand(case.batch, -1, -1, -1)
    outs = []
    with torch.no_grad():
        model.set_counter(0)
        for t in range(case.steps):
            inp = W.unet_inputs(case, t, ucfg)
            to_dev = lambda x: x.to(dev, torch.float16) if x.is_floating_point() else x.to(dev)
            kw = dict(sample=to_dev(inp["sample"]), timestep=inp["timestep"].to(dev).float(),
                      encoder_hidden_states=to_dev(inp["encoder_hidden_states"]))
            if inp["added_cond_kwargs"] is not None:
                kw["added_cond_kwargs"] = {k: to_dev(v) for k, v in inp["added_cond_kwargs"].items()}
            if with_cn:
                kw.update(controlnet_cond=cond, conditioning_scale=scale[t] if isinstance(scale, (list, tuple)) else scale)
            outs.append(model(**kw, return_dict=False)[0].float().cpu().clone())
    return outs


def _close_pipes(pipes, world):
    from torch import distributed as dist
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        for pipe in pipes:
            if pipe.comm_manager is not None:
                pipe.comm_manager.close()
        dist.destroy_process_group()


def _product_unet_worker(rank, case, use_graph, scale, zero, port, outdir):
    _product_init(rank, case, port)
    pipe, ucfg = _product_pipe(case, use_graph, zero)
    outs = _product_steps(pipe, ucfg, case, scale, zero is not None)
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    _close_pipes([pipe], case.world_size)


def _zero_premise_worker(rank, case, port, outdir):
    """Both pipelines in ONE process, so that cuDNN's autotuned algorithms are the same for both."""
    _product_init(rank, case, port)
    plain, ucfg = _product_pipe(case, True, None)
    zero, _ = _product_pipe(case, True, True)
    outs = (_product_steps(plain, ucfg, case, 1.0, False), _product_steps(zero, ucfg, case, 1.0, True))
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    _close_pipes([plain, zero], case.world_size)


def run_zero_premise(case):
    """-> per rank, (outputs without a ControlNet, outputs with a zero-initialised one), CUDA graphs on."""
    from oracle.harness import run_ranks
    return run_ranks(_zero_premise_worker, case)


def run_product_unet(case, use_graph=False, scale=1.0, zero=False):
    """Product UNet + ControlNet per rank and step.  zero=True: a zero-initialised ControlNet; zero=None: no ControlNet at all.
    `scale`: a float, or one per step."""
    from oracle.harness import run_ranks
    return run_ranks(_product_unet_worker, case, use_graph, scale, zero)


def _product_traj_worker(rank, case, num_steps, guidance, port, outdir):
    _product_init(rank, case, port)
    pipe, _ = _product_pipe(case, True)
    image = cond_image(case)
    run = lambda: pipe(prompt="a photo", num_inference_steps=num_steps, guidance_scale=guidance, image=image,
                       controlnet_conditioning_scale=1.0, generator=torch.Generator().manual_seed(case.input_seed)).images
    lat = run()
    lat2 = run()
    torch.cuda.synchronize()
    assert torch.equal(lat, lat2), "second image with the same seed differs from the first"
    torch.save(lat.float().cpu(), os.path.join(outdir, f"rank{rank}.pt"))
    _close_pipes([pipe], case.world_size)


def run_product_trajectory(case, num_steps=8, guidance=5.0):
    from oracle.harness import run_ranks
    return run_ranks(_product_traj_worker, case, num_steps, guidance)
