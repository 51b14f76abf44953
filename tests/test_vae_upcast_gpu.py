"""GPU checks of the upcast VAE decode (DistriAutoencoderKLPP(upcast=True)) and the fp32 kernels it runs.

Kernels: the fp32 GroupNorm (plain, with SiLU, and halo-fused) through DistriGroupNorm over 1, 2 and 3 uneven strips at the
SDXL VAE's up-block shapes against an fp64 GroupNorm of the whole image, one case at magnitude 1e5 with |mean| >> std; the
fp32 halo push / assemble and output gather bit-exactly.
Decode: the full-size SDXL VAE (random weights, force_upcast=True) against an fp64 decode, with test_vae_gpu.py's bar where
B is the compat decoder under diffusers' split (fp16 up to the mid block, fp32 after) on torch's kernels.  The overflow case
scales the up-block resnets' conv2 until the fp64 residual stream passes 1e5: torch's fp16 decode is then non-finite and the
upcast decode still meets the bar.  Split: 2 and 3 ranks on one GPU (DISTRIFUSER_B200_SHARE_GPU=1), 8 GPUs where present.
Pipelines: from_synthetic(..., vae_upcast=True) and the fake diffusers' SDXL decode return the fp32 decode of their latents."""
from __future__ import annotations

import copy
import os
import subprocess
import sys
import tempfile

import pytest
import torch
from torch.nn import functional as F

from helpers import LoopbackArena

pytestmark = pytest.mark.gpu

E_FLOOR, M_FLOOR, E_ABS = 2.0 ** -11, 2.0 ** -9, 2.0 ** -7
F_E, F_M = 1.5, 2.0                      # test_vae_gpu.py's bar
STREAM_MIN = 1e5                         # the overflow case's residual stream, above fp16's 65504


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ================================================================================================================ copies
@pytest.mark.parametrize("up,down", [(-1, 1), (0, 2), (2, -1)])
def test_halo_push_and_assemble_fp32(up, down):
    from distrifuser_b200 import _lib
    L = _lib.lib()
    torch.manual_seed(6)
    b, c, h, w, n = 2, 128, 5, 9, 4
    rank = 1 if up == 0 else (0 if up < 0 else 3)
    row_bytes = w * c * 4
    arena = LoopbackArena(n, [2 * b * row_bytes], rank=rank)
    try:
        x = (torch.randn(b, c, h, w, device="cuda") * 1e5).contiguous(memory_format=torch.channels_last)
        epoch = 7
        arena.set_clock(pub=epoch, rd=epoch)
        _lib.check(L.df_halo_push_dtype(arena.comm, x.data_ptr(), b, h, w, c, 0, arena.tensor_off[0], arena.slot_bytes[0], up, down,
                                        _lib.F32, _stream()), "df_halo_push_dtype")
        torch.cuda.synchronize()
        mine = arena.slot(epoch, 0, rank, 2 * b * row_bytes, torch.float32).view(2, b, w, c)
        xn = x.permute(0, 2, 3, 1)
        if up >= 0:
            assert torch.equal(mine[0], xn[:, 0])
        if down >= 0:
            assert torch.equal(mine[1], xn[:, -1])
        top_src, bot_src = torch.randn(b, w, c, device="cuda"), torch.randn(b, w, c, device="cuda")
        if up >= 0:
            arena.slot(epoch, 0, up, 2 * b * row_bytes, torch.float32).view(2, b, w, c)[1].copy_(top_src)
            arena.flags[0, up] = epoch
        if down >= 0:
            arena.slot(epoch, 0, down, 2 * b * row_bytes, torch.float32).view(2, b, w, c)[0].copy_(bot_src)
            arena.flags[0, down] = epoch
        xp = torch.full((b, c, h + 2, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)
        _lib.check(L.df_halo_assemble_dtype(arena.comm, x.data_ptr(), xp.data_ptr(), b, h, w, c, 0, arena.tensor_off[0],
                                            arena.slot_bytes[0], up, down, 1, _lib.F32, _stream()), "df_halo_assemble_dtype")
        torch.cuda.synchronize()
        xpn = xp.permute(0, 2, 3, 1)
        assert torch.equal(xpn[:, 1:-1], xn)
        assert torch.equal(xpn[:, 0], top_src if up >= 0 else torch.zeros_like(top_src))
        assert torch.equal(xpn[:, -1], bot_src if down >= 0 else torch.zeros_like(bot_src))
    finally:
        arena.close()


def _tiles(H, W, rows, cols):
    return [(0, rows[i], cols[j], 1, rows[i + 1] - rows[i], cols[j + 1] - cols[j])
            for i in range(len(rows) - 1) for j in range(len(cols) - 1)]


# (C, H, W, rects of the 4 ranks, this rank, whether the 16-byte path applies)
GATHER = {
    "vec-col": (3, 8, 16, _tiles(8, 16, [0, 8], [0, 4, 8, 12, 16]), 2, True),          # ws = 4: whole float4 runs
    "scalar-col-ws6": (3, 6, 24, _tiles(6, 24, [0, 6], [0, 6, 12, 18, 24]), 1, False),  # ws = 6: not a multiple of 4
    "scalar-odd-width": (3, 5, 13, _tiles(5, 13, [0, 5], [0, 3, 7, 10, 13]), 3, False),  # W = 13, ws = 3
    "rows-uneven": (3, 11, 8, _tiles(11, 8, [0, 3, 6, 9, 11], [0, 8]), 3, True),       # full width, hs * W = 16: one run
    "rows-odd-run": (3, 7, 5, _tiles(7, 5, [0, 2, 4, 6, 7], [0, 5]), 0, False),        # hs * W = 10: element stores
    "rows-offset-odd": (3, 6, 2, _tiles(6, 2, [0, 2, 3, 5, 6], [0, 2]), 2, False),      # hs * W = 4 but row0 * W = 6
    "image-odd": (3, 7, 3, _tiles(7, 3, [0, 4, 5, 6, 7], [0, 3]), 0, False),           # hs * W = 12 but H * W = 21
}


@pytest.mark.parametrize("name", list(GATHER))
def test_output_gather_2d_fp32(name):
    from distrifuser_b200 import _lib
    Cc, H, W, rects, me, vec = GATHER[name]
    n, E = len(rects), 13
    b0, r0, c0, bs, hs, ws = rects[me]
    full = ws == W
    whole = (hs * W % 4 == 0 and r0 * W % 4 == 0 and H * W % 4 == 0) if full else (ws % 4 == 0 and c0 % 4 == 0 and W % 4 == 0)
    assert whole == vec
    torch.manual_seed(37)
    img = torch.randn(1, Cc, H, W, device="cuda") * 1e5
    nbytes = img.numel() * 4
    arena = LoopbackArena(n, [nbytes], rank=me)
    try:
        arena.clock[2] = E
        for ep in (E + 1, E - 1):
            arena.slot(ep, 0, 0, nbytes, torch.float32).fill_(float("nan"))
        bank = arena.slot(E, 0, 0, nbytes, torch.float32).view(1, Cc, H, W)
        bank.fill_(float("nan"))
        for r, (rb, rr, rc, rbs, rhs, rws) in enumerate(rects):
            if r != me:
                bank[rb:rb + rbs, :, rr:rr + rhs, rc:rc + rws] = img[rb:rb + rbs, :, rr:rr + rhs, rc:rc + rws]
                arena.flags[0, r] = E
        strip = img[b0:b0 + bs, :, r0:r0 + hs, c0:c0 + ws].contiguous()
        out = torch.full_like(img, float("nan"))
        _lib.check(_lib.lib().df_output_gather_2d_dtype(arena.comm, strip.data_ptr(), out.data_ptr(), 1, Cc, H, W, bs, hs, ws, b0,
                                                        r0, c0, 0, arena.tensor_off[0], _lib.F32, _stream()),
                   "df_output_gather_2d_dtype")
        torch.cuda.synchronize()
        assert torch.equal(out, img)
    finally:
        arena.close()


def test_output_gather_fp16_full_width_offset_rows():
    """fp16, full width: hs * W = 8 is one vector, but row0 * W = 12 is not, so the strip goes out in 2-byte stores."""
    from distrifuser_b200 import _lib
    H, W, rects, me, E = 6, 4, _tiles(6, 4, [0, 2, 3, 5, 6], [0, 4]), 2, 5
    b0, r0, c0, bs, hs, ws = rects[me]
    assert hs * W % 8 == 0 and r0 * W % 8 != 0
    img = torch.randn(1, 3, H, W, device="cuda").half()
    nbytes = img.numel() * 2
    arena = LoopbackArena(4, [nbytes], rank=me)
    try:
        arena.clock[2] = E
        bank = arena.slot(E, 0, 0, nbytes).view(1, 3, H, W)
        bank.fill_(float("nan"))
        for r, (rb, rr, rc, rbs, rhs, rws) in enumerate(rects):
            if r != me:
                bank[:, :, rr:rr + rhs] = img[:, :, rr:rr + rhs]
                arena.flags[0, r] = E
        strip = img[:, :, r0:r0 + hs].contiguous()
        out = torch.full_like(img, float("nan"))
        _lib.check(_lib.lib().df_output_gather_2d(arena.comm, strip.data_ptr(), out.data_ptr(), 1, 3, H, W, bs, hs, ws, b0, r0, c0,
                                                  0, arena.tensor_off[0], _stream()), "df_output_gather_2d")
        torch.cuda.synchronize()
        assert torch.equal(out, img)
    finally:
        arena.close()


# ================================================================================================================ GroupNorm
# (name, C, H, W, silu, halo, magnitude): the SDXL VAE's up-block widths at up to 1024^2 pixels
# (the 1e5 cases: local statistics at world 1 without halos, pooled statistics at worlds 2 and 3 with and without)
GN_CASES = [("c512", 512, 128, 128, False, False, 1.0), ("c256-silu", 256, 512, 512, True, False, 1.0),
            ("c128-halo-1024px", 128, 1024, 1024, True, True, 1.0), ("c256-silu-1e5", 256, 128, 128, True, False, 1e5),
            ("c128-halo-1e5", 128, 256, 256, True, True, 1e5)]


def _gn_input(C, H, W, mag):
    """Seeded [1, C, H, W] fp32.  mag > 1: per-channel means near mag with std 0.01 * mag, plus a row gradient so the strips'
    means differ -- E[x^2] / var is ~1e4, the one-pass fp32 formula's failure case."""
    g = torch.Generator(device="cuda").manual_seed(C + H)
    x = torch.randn(1, C, H, W, device="cuda", generator=g)
    if mag > 1:
        ch = 1 + 0.05 * torch.rand(1, C, 1, 1, device="cuda", generator=g)
        x = mag * (ch + 0.01 * x + 0.002 * torch.linspace(-1, 1, H, device="cuda").view(1, 1, H, 1))
    return x


def _gn_worker_cases(cfg, n, r):
    from distrifuser_b200.modules.pp.conv2d import DistriConv2dPP
    from distrifuser_b200.modules.pp.groupnorm import DistriGroupNorm
    from distrifuser_b200.utils import PatchParallelismCommManager, row_offset, split_units
    res = {}
    for name, C, H, W, silu, halo, mag in GN_CASES:
        if halo and n == 1:
            continue                                                 # one rank: no halos
        x = _gn_input(C, H, W, mag)
        torch.manual_seed(C)
        mod = torch.nn.GroupNorm(32, C, eps=1e-6).cuda()
        with torch.no_grad():
            mod.weight.normal_(1, 0.2)
            mod.bias.normal_(0, 0.2)
            ref = F.group_norm(x.double(), 32, mod.weight.double(), mod.bias.double(), 1e-6)
            if silu:
                ref = F.silu(ref)
        units = split_units(H, n)
        lo = row_offset(units, r)
        strip = x[:, :, lo:lo + units[r]].contiguous(memory_format=torch.channels_last)
        ref = ref[:, :, lo:lo + units[r]]
        del x
        gn = DistriGroupNorm(copy.deepcopy(mod), cfg)
        gn.biased_var, gn.fuse_silu, gn.allow_fp32, gn.row_units = True, silu, True, units
        conv = None
        if halo:
            conv = DistriConv2dPP(torch.nn.Conv2d(C, C, 3, padding=1).cuda(), cfg)
            conv.allow_fp32, conv.row_units = True, units
        cm = PatchParallelismCommManager(cfg) if n > 1 else None
        if cm is not None:
            for m in (gn, conv):
                if m is not None:
                    m.set_comm_manager(cm)
            gn(strip)                                                # registration pass
            if conv is not None:
                conv(strip)
            cm.create_buffer()
            cm.step_begin(0)
        with torch.no_grad():
            y = gn(strip, pad_for=conv) if halo else gn(strip)
        torch.cuda.synchronize()
        assert y.dtype == torch.float32
        inner = y[:, :, 1:-1] if halo else y
        err = (inner.double() - ref).abs().max().item()
        rows = (inner[:, :, 0].cpu(), inner[:, :, -1].cpu(), y[:, :, 0].cpu(), y[:, :, -1].cpu()) if halo else None
        res[name] = (err, rows)
        del y, inner, ref, strip
        if cm is not None:
            torch.distributed.barrier()                              # every rank is done with the arenas
            cm.close()
        torch.cuda.empty_cache()
    return res


def _view(world, split_batch=False):
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(height=256, width=256, split_batch=split_batch)
    view = copy.copy(cfg)
    view.n_device_per_batch, view.split_batch, view.mode = cfg.world_size, False, "full_sync"
    return view


def _spawn(fn, world, *args):
    """fn(rank, world, *args) -> picklable, on `world` processes sharing this host's GPUs; -> per-rank results."""
    from torch import multiprocessing as mp

    from oracle.harness import free_port
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, fn, args, free_port(), d), nprocs=world, join=True)
        return [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(world)]


def _worker(rank, world, fn, args, port, outdir):
    from torch import distributed as dist
    if torch.cuda.device_count() < world:
        os.environ["DISTRIFUSER_B200_SHARE_GPU"] = "1"
    os.environ["LOCAL_RANK"] = str(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    out = fn(rank, world, *args)
    torch.save(out, os.path.join(outdir, f"rank{rank}.pt"))
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


def _gn_job(rank, world):
    cfg = _view(world)
    torch.cuda.set_device(cfg.device)
    return _gn_worker_cases(cfg, world, rank)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_groupnorm_fp32_strips(world):
    """Every rank's normalised strip against the fp64 GroupNorm of the whole image (the strips of 3 ranks are uneven:
    128 / 512 / 1024 / 256 rows as 43+43+42 ...); halo-fused: each margin row is the neighbour's boundary row, bit for bit."""
    outs = _spawn(_gn_job, world)
    for name, C, H, W, silu, halo, mag in GN_CASES:
        if halo and world == 1:
            continue
        for r, res in enumerate(outs):
            err, rows = res[name]
            print(f"{name} world {world} rank {r}: max |err| {err:.3e}")
            assert err < 2e-4, f"{name} rank {r}: max |err| {err:.3e} against fp64"
            if halo:
                first, last, top, bottom = rows
                assert torch.equal(top, outs[r - 1][name][1][1] if r > 0 else torch.zeros_like(top)), f"{name} rank {r} top"
                assert torch.equal(bottom, outs[r + 1][name][1][0] if r < world - 1 else torch.zeros_like(bottom)), \
                    f"{name} rank {r} bottom"


# ================================================================================================================ decode
def _vae(scale=None, device="cuda"):
    """The full-size SDXL VAE (force_upcast=True) under a fixed seed, fp32; `scale`: the up-block resnets' conv2 (weight and
    bias) multiplied by it."""
    from distrifuser_b200.compat.vae import SDXL_VAE, AutoencoderKL
    torch.manual_seed(11)
    vae = AutoencoderKL(**SDXL_VAE).to(device).eval()
    if scale is not None:
        with torch.no_grad():
            for blk in vae.decoder.up_blocks:
                for res in blk.resnets:
                    res.conv2.weight.mul_(scale)
                    res.conv2.bias.mul_(scale)
    return vae


def _latent(rows, cols):
    g = torch.Generator().manual_seed(5)
    return torch.randn(1, 4, rows, cols, generator=g).to("cuda", torch.float16)


def _stream_max(vae, z):
    """max |x| over the outputs of the up blocks' resnets (the residual stream) in an fp64 decode, and that decode."""
    peak = [0.0]
    hooks = [res.register_forward_hook(lambda m, i, o: peak.__setitem__(0, max(peak[0], o.abs().max().item())))
             for blk in vae.decoder.up_blocks for res in blk.resnets]
    try:
        with torch.no_grad():
            out = vae.decode(z.double()).sample
    finally:
        for h in hooks:
            h.remove()
    return peak[0], out


_SCALE: dict = {}


def _overflow_scale():
    """conv2 scale that takes the fp64 residual stream of a 64 x 48 latent to ~3e5: the resnets' branches grow linearly with it
    (the GroupNorms cancel every other scale); the mid block's part of the stream does not, hence a few rounds."""
    if "s" not in _SCALE:
        s = 1.0
        for _ in range(4):
            peak, _ = _stream_max(_vae(s).double(), _latent(64, 48))
            if peak > 2 * STREAM_MIN:
                break
            s *= 3 * STREAM_MIN / peak
        _SCALE["s"] = s
        torch.cuda.empty_cache()
    return _SCALE["s"]


def _split_reference(vae):
    """The compat decoder (no wrappers) under diffusers' upcast split, on torch's kernels."""
    from distrifuser_b200.models.distri_vae_pp import apply_upcast_split
    b = copy.deepcopy(vae)
    apply_upcast_split(b)
    return b


_REF: dict = {}


def _reference(rows, cols, overflow):
    """(fp64 decode, B = torch's decode under the upcast split) of the seeded VAE and latent, computed once per case; the
    overflow case also asserts the fp64 stream and that torch's fp16 decode is non-finite."""
    key = (rows, cols, overflow)
    if key not in _REF:
        scale = _overflow_scale() if overflow else None
        vae = _vae(scale)
        z = _latent(rows, cols)
        peak, r = _stream_max(copy.deepcopy(vae).double(), z)
        if overflow:
            assert peak > STREAM_MIN, f"fp64 residual stream peaks at {peak:.3e}"
            with torch.no_grad():
                fp16 = copy.deepcopy(vae).half().decode(z).sample
            assert not torch.isfinite(fp16).all(), "torch's fp16 decode should overflow"
            del fp16
        with torch.no_grad():
            b = _split_reference(vae).decode(z).sample.double()
        _REF[key] = (r, b, scale)
        del vae
        torch.cuda.empty_cache()
    return _REF[key]


def _metrics(x, ref):
    d = (x.double() - ref).flatten()
    rms = ref.pow(2).mean().sqrt()
    return (d.norm() / ref.flatten().norm()).item(), (d.abs().max() / rms).item()


def _check(name, got, rows, cols, overflow=False):
    r, b, _ = _reference(rows, cols, overflow)
    assert got.dtype == torch.float32 and got.shape == r.shape and torch.isfinite(got).all(), name
    e_p, m_p = _metrics(got, r)
    e_b, m_b = _metrics(b, r)
    print(f"{name}: e_P {e_p:.3e} e_B {e_b:.3e} m_P {m_p:.3e} m_B {m_b:.3e}")
    assert e_p <= F_E * e_b + E_FLOOR and m_p <= F_M * m_b + M_FLOOR and e_p < E_ABS, \
        f"{name}: e_P {e_p:.3e} (torch split {e_b:.3e}), m_P {m_p:.3e} (torch split {m_b:.3e})"


@pytest.mark.parametrize("px", [512, 1024])
def test_decode_upcast_world1_vs_fp64(px):
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    from distrifuser_b200.utils import DistriConfig
    rows = cols = px // 8
    pp = DistriAutoencoderKLPP(_vae().half(), DistriConfig(height=px, width=px), upcast=True)
    z = _latent(rows, cols)
    got = pp.decode(z).sample
    assert torch.equal(got, pp.decode(z, return_dict=False)[0])
    _check(f"sdxl upcast {px}^2 world 1", got, rows, cols)


def test_decode_upcast_overflow_world1():
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    from distrifuser_b200.utils import DistriConfig
    _, _, scale = _reference(64, 48, True)
    pp = DistriAutoencoderKLPP(_vae(scale), DistriConfig(height=512, width=384), upcast=True)
    _check("sdxl upcast overflow 64x48 world 1", pp.decode(_latent(64, 48)).sample, 64, 48, overflow=True)


def _decode_job(rank, world, cases, default_cfg):
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    from distrifuser_b200.utils import DistriConfig
    imgs = []
    for rows, cols, scale in cases:
        kw = {} if default_cfg else dict(split_batch=False)
        cfg = DistriConfig(height=8 * rows, width=8 * cols, **kw)    # selects this rank's device before anything is built
        torch.cuda.set_device(cfg.device)
        pp = DistriAutoencoderKLPP(_vae(scale), cfg, upcast=True)
        z = _latent(rows, cols)
        img = pp.decode(z).sample.clone()
        assert torch.equal(img, pp.decode(z).sample), f"rank {rank}: the second decode differs"
        imgs.append(img.cpu())
        torch.cuda.synchronize()
        torch.distributed.barrier()
        pp.close()
        del pp
        torch.cuda.empty_cache()
    return imgs


def _check_split(world, shapes, default_cfg=False):
    cases = [(rows, cols, _reference(rows, cols, ov)[2]) for rows, cols, ov in shapes]
    outs = _spawn(_decode_job, world, cases, default_cfg)
    for k, (rows, cols, ov) in enumerate(shapes):
        imgs = [o[k] for o in outs]
        for r, img in enumerate(imgs):
            assert torch.equal(img, imgs[0]), f"rank {r} holds another image"
        _check(f"sdxl upcast split over {world}, latent {rows}x{cols}{' overflow' if ov else ''}", imgs[0].cuda(), rows, cols, ov)


@pytest.mark.parametrize("world", [2, 3], ids=["n2", "n3-uneven"])
def test_split_decode_upcast_share_gpu(world):
    _check_split(world, [(64, 48, False), (64, 48, True)], default_cfg=world == 2)


def test_split_decode_upcast_eight_gpus():
    if torch.cuda.device_count() < 8:
        pytest.skip("needs 8 GPUs")
    _check_split(8, [(128, 128, False), (64, 48, True)])


# ================================================================================================================ pipelines
def test_from_synthetic_vae_upcast_pt_output():
    from oracle import workloads as W
    from distrifuser_b200.compat.vae import SDXL_VAE, AutoencoderKL
    from distrifuser_b200.pipelines import DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(height=256, width=192, use_cuda_graph=False)
    torch.manual_seed(3)
    vae = AutoencoderKL(**SDXL_VAE)
    pipe = DistriSDXLPipeline.from_synthetic(cfg, unet_config=W.unet_config("tiny_sdxl"), vae=vae, vae_upcast=True)
    run = lambda **kw: pipe(prompt="a photo", num_inference_steps=3, guidance_scale=5.0,
                            generator=torch.Generator().manual_seed(1), **kw).images
    lat = run()
    img = run(output_type="pt")
    with torch.no_grad():
        dec = pipe.pipeline.vae.decode((lat / SDXL_VAE["scaling_factor"]).half()).sample
    assert dec.dtype == torch.float32 and img.dtype == torch.float32
    assert img.shape == (1, 3, 256, 192) and img.min() >= 0 and img.max() <= 1
    assert torch.equal(img, (dec / 2 + 0.5).clamp(0, 1))
    assert torch.equal(run(), lat)


def test_fake_diffusers_sdxl_upcast_decode():
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "run_from_pretrained_vae_upcast.py"), "gpu"], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "OK from_pretrained vae_upcast gpu" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
