"""TEST INFRASTRUCTURE (oracle) -- multi-rank CPU driver (gloo) for the parity workloads.

`impl="oracle"`    runs the restatement in oracle/pp_modules.py (works anywhere).
`impl="reference"` runs the UNMODIFIED reference modules imported from /root/reference through the
                   diffusers stub (only possible in the build container; used by oracle/make_golden.py).
The UNet drivers serve every UNet case type: patch parallelism on equal (UNetCase) or uneven (RaggedCase) row strips, and
naive patch (naive_patch.NaiveCase); the case's config_kwargs() choose the wrapper.  With `controlnet=` they run UNet +
ControlNet (ControlledUNet) under the same patch-parallel wrapper, whose surgery wraps both models' layers alike.
Both follow the reference's own bring-up order (pipelines.py:131-145): registration pass, create buffers,
pre-run pass, then `set_counter(0)` and the denoising calls (pipelines.py:57).
"""
from __future__ import annotations

import os
import socket
import sys
import tempfile

import torch
from torch import distributed as dist
from torch import multiprocessing as mp
from torch import nn
from torch.nn import functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
STUB = os.path.join(HERE, "diffusers_stub")
REFERENCE = "/root/reference"


def _paths(impl):
    for p in (STUB, os.path.dirname(HERE)):
        if p not in sys.path:
            sys.path.insert(0, p)
    if impl == "reference":
        if not os.path.isdir(REFERENCE):
            raise RuntimeError("the reference tree is only available in the build container")
        if REFERENCE not in sys.path:
            sys.path.insert(0, REFERENCE)


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _init(rank, world, port):
    # tiny parity workloads: more than ~16 OpenMP threads only adds synchronisation overhead (64-thread hosts ran 10x slower)
    torch.set_num_threads(max(1, min(16, (os.cpu_count() or 8) // world)))
    if world > 1:
        dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")


def _groups(cfg):
    """batch_group construction of DistriConfig (utils.py:84-96)."""
    if cfg.do_classifier_free_guidance and cfg.split_batch and cfg.world_size >= 2:
        half = cfg.world_size // 2
        groups = [dist.new_group(list(range(i * half, (i + 1) * half))) for i in range(2)]
        cfg.batch_group = groups[cfg.batch_idx()]


# ---------------------------------------------------------------------------------------------- chain
class _Chain(nn.Module):
    """GroupNorm -> SiLU -> 3x3 conv -> tokens -> self-attention -> cross-attention."""

    def __init__(self, case, w):
        super().__init__()
        from diffusers.models.attention_processor import Attention
        C = case.C
        self.norm = nn.GroupNorm(case.groups, C, eps=1e-5)
        self.conv = nn.Conv2d(C, C, 3, stride=case.stride, padding=1)
        self.attn1 = Attention(C, None, case.heads, C // case.heads)
        self.attn2 = Attention(C, case.cross_dim, case.heads, C // case.heads)
        with torch.no_grad():
            self.norm.weight.copy_(w["gn_w"]); self.norm.bias.copy_(w["gn_b"])
            self.conv.weight.copy_(w["conv_w"]); self.conv.bias.copy_(w["conv_b"])
            for a, p in ((self.attn1, ("wq", "wk", "wv", "wo", "bo")), (self.attn2, ("xq", "xk", "xv", "xo", "xbo"))):
                a.to_q.weight.copy_(w[p[0]]); a.to_k.weight.copy_(w[p[1]]); a.to_v.weight.copy_(w[p[2]])
                a.to_out[0].weight.copy_(w[p[3]]); a.to_out[0].bias.copy_(w[p[4]])

    def forward(self, x, ehs):
        y_gn = self.norm(x)
        y_conv = self.conv(F.silu(y_gn))
        b, c, h, w = y_conv.shape
        tok = y_conv.permute(0, 2, 3, 1).reshape(b, h * w, c)
        y_sa = self.attn1(tok)
        y_ca = self.attn2(y_sa, encoder_hidden_states=ehs)
        return y_gn, y_conv, y_sa, y_ca


def _chain_worker(rank, case, impl, port, outdir):
    _paths(impl)
    from oracle import workloads as W
    _init(rank, case.n, port)
    cfg = W.DuckConfig(case.n, rank, height=8 * case.H, width=8 * case.W, do_classifier_free_guidance=False,
                       warmup_steps=case.warmup_steps, comm_checkpoint=2, mode=case.mode)
    chain = _Chain(case, W.chain_weights(case)).eval()
    if impl == "reference":
        from distrifuser.modules.pp.attn import DistriCrossAttentionPP, DistriSelfAttentionPP
        from distrifuser.modules.pp.conv2d import DistriConv2dPP
        from distrifuser.modules.pp.groupnorm import DistriGroupNorm
        from distrifuser.utils import PatchParallelismCommManager
        chain.norm = DistriGroupNorm(chain.norm, cfg)
        chain.conv = DistriConv2dPP(chain.conv, cfg)
        chain.attn1 = DistriSelfAttentionPP(chain.attn1, cfg)
        chain.attn2 = DistriCrossAttentionPP(chain.attn2, cfg)
        mods = [chain.norm, chain.conv, chain.attn1, chain.attn2]
        comm = PatchParallelismCommManager(cfg)
        begin, set_comm = (lambda: None), (lambda m: m.set_comm_manager(comm))
        create = lambda: comm.create_buffer()
    else:
        from oracle import pp_modules as P
        chain.norm = P.OracleGroupNorm(chain.norm, cfg)
        chain.conv = P.OracleConv2d(chain.conv, cfg)
        chain.attn1 = P.OracleSelfAttention(chain.attn1, cfg)
        chain.attn2 = P.OracleCrossAttention(chain.attn2, cfg)
        mods = [chain.norm, chain.conv, chain.attn1, chain.attn2]
        comm = P.OracleComm(cfg)
        begin, set_comm = comm.begin_step, (lambda m: m.set_comm(comm))
        create = lambda: comm.create()
    rows = case.H // case.n
    local = lambda x: x[:, :, rank * rows:(rank + 1) * rows].contiguous()
    outs = []
    with torch.no_grad():
        x0, ehs = W.chain_input(case, 0)
        for m in mods:
            set_comm(m)
        chain(local(x0), ehs)          # registration pass (pipelines.py:138-139)
        create()                       # pipelines.py:140-141
        for m in mods:
            m.set_counter(0)
        chain(local(x0), ehs)          # pre-run (pipelines.py:144-145)
        for m in mods:
            m.set_counter(0)           # pipelines.py:57
        for t in range(case.steps):
            x, ehs = W.chain_input(case, t)
            if impl == "oracle" and comm.slots is not None:
                begin()
            outs.append(tuple(o.clone() for o in chain(local(x), ehs)))
        if impl == "reference":
            comm.clear()
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    if case.n > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_chain(case, impl="oracle"):
    """-> outs[rank][step] = (y_gn, y_conv, y_selfattn, y_crossattn) for that rank's row strip."""
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_chain_worker, args=(case, impl, free_port(), d), nprocs=case.n, join=True)
        return [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(case.n)]


# ---------------------------------------------------------------------------------------------- UNet
def _unet_config(case, rank):
    """DuckConfig of a UNet case (patch, naive patch or uneven strips) on `rank`, its batch groups made."""
    from oracle import workloads as W
    cfg = W.DuckConfig(case.world_size, rank, **case.config_kwargs())
    if case.world_size > 1:
        _groups(cfg)
    return cfg


class ControlledUNet(nn.Module):
    """Runs ControlNet then UNet with the UNet's call signature; the conditioning image `cond` (batch 1) is shared by both CFG
    branches.  `down_blocks` is the UNet's, so that OracleUNetPP derives the row plan from it."""

    def __init__(self, unet, controlnet, cond, scale=1.0):
        super().__init__()
        self.unet, self.controlnet, self.cond, self.scale = unet, controlnet, cond, scale

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
        return self.unet(sample, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs,
                         down_block_additional_residuals=down, mid_block_additional_residual=mid, return_dict=False)


def _check_controlnet(case, impl, controlnet):
    if controlnet is not None and impl == "reference":
        raise ValueError("the reference has no ControlNet: a ControlNet case runs on impl='oracle' only")
    if controlnet is not None and case.config_kwargs().get("parallelism") == "naive_patch":
        raise NotImplementedError("a ControlNet runs under patch parallelism only (parallelism='patch')")


def _unet(case, controlnet=None, scale=1.0):
    """The seeded UNet of the case, or with `controlnet` the UNet + ControlNet module: "drawn" is the seeded ControlNet with
    its zero-initialised layers drawn (non-zero residuals), "zero" the one as initialised."""
    from oracle import workloads as W
    unet = W.make_unet(case.family, case.weight_seed)
    if controlnet is None:
        return unet
    cn = W.make_controlnet(case.family, case.weight_seed, zero=controlnet == "zero")
    return ControlledUNet(unet, cn, W.cond_image(case), scale)


def _oracle_unet(unet, cfg, bessel=True):
    from oracle import pp_modules as P
    if cfg.parallelism == "naive_patch":
        from oracle.naive_patch import OracleNaivePatchUNet
        return OracleNaivePatchUNet(unet, cfg)
    return P.OracleUNetPP(unet, cfg, bessel=bessel)


def _unet_worker(rank, case, impl, bessel, row_units, controlnet, scale, port, outdir):
    _paths(impl)
    from oracle import workloads as W
    _init(rank, case.world_size, port)
    cfg = _unet_config(case, rank)
    ucfg = W.unet_config(case.family)
    unet = _unet(case, controlnet, scale)
    first = W.unet_inputs(case, 0, ucfg)
    outs = []
    with torch.no_grad():
        if impl == "reference":
            from distrifuser.utils import PatchParallelismCommManager
            if cfg.parallelism == "naive_patch":
                from distrifuser.models.naive_patch_sdxl import NaivePatchUNet as Model
            else:
                from distrifuser.models.distri_sdxl_unet_pp import DistriUNetPP as Model
            model = Model(unet, cfg)
            comm = None
            if cfg.n_device_per_batch > 1:                                   # pipelines.py:131-141
                comm = PatchParallelismCommManager(cfg)
                model.set_comm_manager(comm)
                model.set_counter(0)
                model(**first, return_dict=False, record=True)
                if comm.numel > 0:                                            # naive patch registers nothing
                    comm.create_buffer()
            model.set_counter(0)
            model(**first, return_dict=False, record=True)                    # pipelines.py:144-145
            model.set_counter(0)                                              # pipelines.py:57
            for t in range(case.steps):
                outs.append(model(**W.unet_inputs(case, t, ucfg), return_dict=False)[0].clone())
            if comm is not None:
                comm.clear()
        else:
            model = _oracle_unet(unet, cfg, bessel)
            if row_units is not None:
                assert model.units == row_units, f"oracle row plan {model.units}, expected {row_units}"
            model.prepare(first)
            model.set_counter(0)
            for t in range(case.steps):
                outs.append(model(**W.unet_inputs(case, t, ucfg)).clone())
    torch.save(outs, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(worker, case, *args):
    """Runs worker(rank, case, *args, port, outdir) on every rank -> what each rank saved."""
    with tempfile.TemporaryDirectory() as d:
        if case.world_size == 1:
            worker(0, case, *args, 0, d)
        else:
            mp.spawn(worker, args=(case, *args, free_port(), d), nprocs=case.world_size, join=True)
        return [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(case.world_size)]


def run_unet(case, impl="oracle", bessel=True, row_units=None, controlnet=None, scale=1.0):
    """-> outs[step] = eps prediction [B,4,H,W] (asserted identical on every rank).  The case picks the UNet wrapper: patch
    parallelism (UNetCase, RaggedCase) or naive patch (NaiveCase).  `bessel=False` drops the oracle GroupNorm's local-count
    Bessel factor; `row_units`, when given, is asserted to be the oracle's row plan.  `controlnet` ("drawn" or "zero", see
    _unet) runs UNet + ControlNet at conditioning scale `scale` on the case's conditioning image (workloads.cond_image)."""
    _check_controlnet(case, impl, controlnet)
    per_rank = run_ranks(_unet_worker, case, impl, bessel, row_units, controlnet, scale)
    for r in range(1, case.world_size):
        for a, b in zip(per_rank[0], per_rank[r]):
            assert torch.equal(a, b), "final output must be identical on all ranks (distri_sdxl_unet_pp.py:166-168)"
    return per_rank[0]


# ---------------------------------------------------------------------------------------------- denoising trajectory
class _OracleUNetAdapter:
    """Gives an oracle UNet wrapper the call signature the latent pipeline uses (unet(x, t, encoder_hidden_states=...)[0])."""

    def __init__(self, model, config):
        self.model, self.config = model, config

    def set_counter(self, c):
        self.model.set_counter(c)

    def __call__(self, sample, timestep, encoder_hidden_states=None, added_cond_kwargs=None, return_dict=False):
        t = timestep
        if torch.is_tensor(t) and t.ndim == 0:
            t = t.expand(sample.shape[0])
        return (self.model(sample, t, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs),)


def _traj_worker(rank, case, num_steps, guidance, controlnet, port, outdir):
    _paths("oracle")
    from oracle import workloads as W
    from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline      # the denoising loop itself is shared code:
    _init(rank, case.world_size, port)                                       # only the UNet path differs between the arms
    cfg = _unet_config(case, rank)
    ucfg = W.unet_config(case.family)
    unet = _unet(case, controlnet)
    model = _oracle_unet(unet, cfg)
    model.prepare(W.unet_inputs(case, 0, ucfg))
    pipe = SyntheticLatentPipeline(_OracleUNetAdapter(model, unet.config), sdxl=ucfg.get("addition_embed_type") == "text_time",
                                   device="cpu", dtype=torch.float32)
    model.set_counter(0)
    g = torch.Generator().manual_seed(case.input_seed)
    with torch.no_grad():
        lat = pipe(prompt="a photo", height=cfg.height, width=cfg.width, num_inference_steps=num_steps,
                   guidance_scale=guidance, generator=g).images
    torch.save(lat, os.path.join(outdir, f"rank{rank}.pt"))
    if case.world_size > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_trajectory(case, num_steps=8, guidance=5.0, controlnet=None):
    """Final latents of a `num_steps` Euler trajectory with the ORACLE UNet path (fp32 CPU) -> [1,4,H,W].  `controlnet` as
    in run_unet, at scale 1."""
    _check_controlnet(case, "oracle", controlnet)
    outs = run_ranks(_traj_worker, case, num_steps, guidance, controlnet)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    return outs[0]
