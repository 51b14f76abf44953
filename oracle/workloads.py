"""TEST INFRASTRUCTURE (oracle) -- seeded synthetic workloads shared by the golden-vector generator
(oracle/make_golden.py, runs the REAL reference), the oracle restatement (oracle/pp_modules.py) and the
GPU parity tests.  Everything is regenerated from integer seeds so fixtures only store outputs.

Inputs follow SURVEY.md 8(d): sample = randn([B,4,S,T]) (S = T but for the uneven-strip cases);
encoder_hidden_states = randn([B,77,cross]); text_embeds = randn([B,pooled]); time_ids = [H,W,0,0,H,W]
(reference: pipelines.py:73-75,106-112).
"""
from __future__ import annotations

import dataclasses
from types import SimpleNamespace

import torch
from torch.nn import functional as F

MODES = ("corrected_async_gn", "stale_gn", "sync_gn", "separate_gn", "full_sync", "no_sync")


class DuckConfig:
    """Duck-typed stand-in for the reference's DistriConfig, which cannot be constructed on CPU because it
    hard-codes ``init_process_group("nccl")`` and ``torch.cuda.set_device`` (utils.py:40,80-81).
    Field and method semantics restated from utils.py:52-110."""

    def __init__(self, world_size, rank, *, height, width, do_classifier_free_guidance=True, split_batch=True,
                 warmup_steps=4, comm_checkpoint=60, mode="corrected_async_gn", parallelism="patch", split_scheme="row",
                 batch_group=None, device="cpu"):
        self.world_size, self.rank = world_size, rank
        self.height, self.width = height, width
        self.do_classifier_free_guidance = do_classifier_free_guidance
        self.split_batch = split_batch
        self.warmup_steps, self.comm_checkpoint, self.mode = warmup_steps, comm_checkpoint, mode
        self.use_cuda_graph = False
        self.parallelism, self.split_scheme, self.verbose = parallelism, split_scheme, False
        if do_classifier_free_guidance and split_batch:          # utils.py:68-75
            n = world_size // 2
            if n == 0:
                n = 1
        else:
            n = world_size
        self.n_device_per_batch = n
        self.device = torch.device(device)
        self.batch_group = batch_group
        self.split_group = None

    def batch_idx(self, rank=None):                              # utils.py:98-104
        rank = self.rank if rank is None else rank
        if self.do_classifier_free_guidance and self.split_batch:
            return 1 - int(rank < (self.world_size // 2))
        return 0

    def split_idx(self, rank=None):                              # utils.py:106-109
        rank = self.rank if rank is None else rank
        return rank % self.n_device_per_batch


class _PatchCase:
    """What the drivers read from a patch-parallel case beyond its fields.  Methods and properties, not fields: the golden
    fixtures pin each case type's fields (`gold["case"] == case.__dict__`)."""

    @property
    def batch(self):
        return 2 if self.cfg else 1

    def config_kwargs(self) -> dict:
        """Keywords of DistriConfig (and of the oracle's DuckConfig) for this case."""
        H, W = self.hw
        return dict(height=8 * H, width=8 * W, do_classifier_free_guidance=self.cfg, split_batch=self.split_batch,
                    warmup_steps=self.warmup_steps, comm_checkpoint=self.comm_checkpoint, mode=self.mode)


@dataclasses.dataclass(frozen=True)
class UNetCase(_PatchCase):
    """One end-to-end tiny-UNet parity case."""
    name: str
    family: str = "tiny_sdxl"        # tiny_sdxl | tiny_sd15
    world_size: int = 2
    cfg: bool = True                 # do_classifier_free_guidance
    split_batch: bool = True
    mode: str = "corrected_async_gn"
    warmup_steps: int = 1
    steps: int = 4
    latent: int = 32                 # latent side S (image side = 8*S)
    comm_checkpoint: int = 20        # <= registered tensors in every mode (SURVEY D-13): every module sees 1-step-stale data, as in SDXL / SD1.x
    weight_seed: int = 0
    input_seed: int = 1234

    @property
    def hw(self):
        """Latent rows and columns (image side / 8)."""
        return self.latent, self.latent


UNET_CASES = (
    UNetCase("sdxl_w1", world_size=1),                               # config-1 shaped plumbing case, world 1
    UNetCase("sdxl_w2_nosplit", world_size=2, split_batch=False),    # n=2, b=2
    UNetCase("sdxl_w4_split", world_size=4),                         # n=2, b=1 (CFG halves)
    UNetCase("sdxl_w4_nosplit", world_size=4, split_batch=False),    # n=4, b=2
    UNetCase("sdxl_w2_fullsync", world_size=2, split_batch=False, mode="full_sync"),
    UNetCase("sdxl_w2_stale", world_size=2, split_batch=False, mode="stale_gn"),
    UNetCase("sdxl_w2_nosync", world_size=2, split_batch=False, mode="no_sync"),
    UNetCase("sdxl_w2_syncgn", world_size=2, split_batch=False, mode="sync_gn"),
    UNetCase("sdxl_w2_sepgn", world_size=2, split_batch=False, mode="separate_gn"),
    UNetCase("sd15_w2_nosplit", family="tiny_sd15", world_size=2, split_batch=False, mode="stale_gn"),
    UNetCase("sdxl_w8_split", world_size=8),                          # n=4, b=1
    UNetCase("sd15_w4_nosplit", family="tiny_sd15", world_size=4, split_batch=False, mode="stale_gn"),   # n=4, b=2; d=40/80/160
    UNetCase("sd15_w8_split", family="tiny_sd15", world_size=8),      # n=4, b=1, corrected_async_gn (BASELINE configs[4] layout)
)


@dataclasses.dataclass(frozen=True)
class RaggedCase(_PatchCase):
    """A patch-parallel case at a latent of lat_h x lat_w, where the patch count need not divide the latent height into
    equal strips (the reference asserts equal strips, so these cases have no reference goldens)."""
    name: str
    family: str = "tiny_sdxl"
    world_size: int = 2
    cfg: bool = True
    split_batch: bool = False
    mode: str = "corrected_async_gn"
    warmup_steps: int = 1
    steps: int = 4
    lat_h: int = 36                  # latent rows (image height / 8)
    lat_w: int = 28
    comm_checkpoint: int = 20
    weight_seed: int = 0
    input_seed: int = 4321

    @property
    def hw(self):
        return self.lat_h, self.lat_w


def unet_config(family: str) -> dict:
    from diffusers.models.unet_2d_condition import (sd15_config, sdxl_config, tiny_sd15_config,
                                                    tiny_sdxl_config)
    return {"tiny_sdxl": tiny_sdxl_config, "tiny_sd15": tiny_sd15_config, "sdxl": sdxl_config,
            "sd15": sd15_config}[family]()


def make_unet(family: str, seed: int = 0, dtype=torch.float32):
    """Random-weight UNet: torch default init under manual_seed(seed) (SURVEY 8d)."""
    from diffusers.models.unet_2d_condition import UNet2DConditionModel
    torch.manual_seed(seed)
    unet = UNet2DConditionModel(**unet_config(family))
    return unet.to(dtype).eval()


def make_controlnet(family: str, seed: int = 0, zero: bool = False, dtype=torch.float32):
    """Seeded ControlNet.  zero=False also draws the zero-initialised layers (the conditioning network's conv_out and the
    1x1 zero convs), so that the residuals are not zero and the parity tests see them."""
    from diffusers.models.controlnet import ControlNetModel
    torch.manual_seed(seed + 101)
    cn = ControlNetModel(**unet_config(family))
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


def unet_inputs(case, step: int, cfg_dict: dict, dtype=torch.float32):
    """Inputs of denoise call `step` (full CFG batch, as the diffusers loop hands them to the UNet) at the case's latent."""
    g = torch.Generator().manual_seed(case.input_seed + 7919 * step)
    B, (S, T) = case.batch, case.hw
    sample = torch.randn(B, 4, S, T, generator=g)
    g2 = torch.Generator().manual_seed(case.input_seed)            # prompt embeddings are constant per image
    ehs = torch.randn(B, 77, cfg_dict["cross_attention_dim"], generator=g2)
    timestep = torch.full((B,), 981 - 20 * step, dtype=torch.long)
    added = None
    if cfg_dict.get("addition_embed_type") == "text_time":
        pooled = cfg_dict["projection_class_embeddings_input_dim"] - 6 * cfg_dict["addition_time_embed_dim"]
        text = torch.randn(B, pooled, generator=g2)
        H, W = float(8 * S), float(8 * T)
        ids = torch.tensor([[H, W, 0.0, 0.0, H, W]] * B)
        added = {"text_embeds": text.to(dtype), "time_ids": ids.to(dtype)}
    return dict(sample=sample.to(dtype), timestep=timestep, encoder_hidden_states=ehs.to(dtype),
                added_cond_kwargs=added)


# ---------------------------------------------------------------- module-chain cases (GN -> conv -> self-attn -> cross-attn)
@dataclasses.dataclass(frozen=True)
class ChainCase:
    name: str
    n: int = 2                 # patch ranks (world == n, no CFG split)
    mode: str = "corrected_async_gn"
    b: int = 1
    C: int = 64
    heads: int = 1
    groups: int = 8
    H: int = 16                # full height of the activation
    W: int = 12
    stride: int = 1
    warmup_steps: int = 1
    steps: int = 4
    seed: int = 99
    cross_dim: int = 32


CHAIN_CASES = tuple(
    [ChainCase(f"chain_n2_{m}", n=2, mode=m) for m in MODES]
    + [ChainCase("chain_n4_corrected", n=4, b=2, C=128, heads=2, groups=32, H=16, W=8),
       ChainCase("chain_n4_stride2", n=4, stride=2, H=32, W=8, mode="full_sync"),
       ChainCase("chain_n8_corrected", n=8, H=32, W=4)]
)


def chain_weights(case: ChainCase):
    g = torch.Generator().manual_seed(case.seed)
    C = case.C
    r = lambda *s: torch.randn(*s, generator=g)
    return dict(
        gn_w=1 + 0.1 * r(C), gn_b=0.1 * r(C),
        conv_w=r(C, C, 3, 3) / (3 * C ** 0.5), conv_b=0.1 * r(C),
        wq=r(C, C) / C ** 0.5, wk=r(C, C) / C ** 0.5, wv=r(C, C) / C ** 0.5, wo=r(C, C) / C ** 0.5, bo=0.1 * r(C),
        xq=r(C, C) / C ** 0.5, xk=r(C, case.cross_dim) / case.cross_dim ** 0.5,
        xv=r(C, case.cross_dim) / case.cross_dim ** 0.5, xo=r(C, C) / C ** 0.5, xbo=0.1 * r(C),
    )


def chain_input(case: ChainCase, step: int):
    """Full-height activation of step `step` ([b,C,H,W]); rank r owns rows [r*H/n,(r+1)*H/n)."""
    g = torch.Generator().manual_seed(case.seed * 31 + step)
    x = torch.randn(case.b, case.C, case.H, case.W, generator=g) * (1.0 + 0.25 * step) + 0.3 * step
    ehs = torch.randn(case.b, 7, case.cross_dim, generator=torch.Generator().manual_seed(case.seed + 5))
    return x, ehs
