"""GPU parity of the patch-parallel VAE decode (DistriAutoencoderKLPP).

World 1: the product's decode of the full-size SD1.x and SDXL VAE decoders (random weights under a fixed seed; SDXL's with
force_upcast=False) against the compat decoder run in fp64, with the bar of test_layer_parity_gpu.py applied to the image:
with e = |X - R|_2 / |R|_2 and m = max|X - R| / rms(R), R the fp64 decode and X = P (the product) or B (the compat decoder
in fp16 on torch's kernels),  e_P <= F_E * e_B + 2^-11,  m_P <= F_M * m_B + 2^-9,  e_P < 2^-7.
Split: 2 and 3 ranks on one GPU (DISTRIFUSER_B200_SHARE_GPU=1), and 8 GPUs where present, against the same fp64 decode with
the same bar, every rank holding the same image.  Pipeline: from_synthetic(..., vae=...) with output_type="pt" is the decode
of the latents it returns."""
from __future__ import annotations

import copy
import os
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

E_FLOOR, M_FLOOR, E_ABS = 2.0 ** -11, 2.0 ** -9, 2.0 ** -7
F_E, F_M = 1.5, 2.0          # the whole decoder as one module; the same order as the UNet's factors in test_layer_parity_gpu.py


def _vae(family, dtype=torch.float16, device="cuda"):
    from distrifuser_b200.compat.vae import SD15_VAE, SDXL_VAE, AutoencoderKL
    cfg = SD15_VAE if family == "sd15" else dict(SDXL_VAE, force_upcast=False)
    torch.manual_seed(11)
    return AutoencoderKL(**cfg).to(device, dtype).eval()


def _latent(rows, cols):
    g = torch.Generator().manual_seed(5)
    return torch.randn(1, 4, rows, cols, generator=g).to("cuda", torch.float16)


def _metrics(x, ref):
    d = (x.double() - ref).flatten()
    rms = ref.pow(2).mean().sqrt()
    return (d.norm() / ref.flatten().norm()).item(), (d.abs().max() / rms).item()


_REF: dict = {}


def _reference(family, rows, cols):
    """(fp64 decode, torch fp16 decode) of the seeded decoder and latent, computed once per shape."""
    key = (family, rows, cols)
    if key not in _REF:
        vae = _vae(family)
        z = _latent(rows, cols)
        with torch.no_grad():
            b = vae.decode(z).sample.double()
            r = copy.deepcopy(vae).double().decode(z.double()).sample
        _REF.clear()
        _REF[key] = (r, b)
        del vae
        torch.cuda.empty_cache()
    return _REF[key]


def _check(name, got, family, rows, cols):
    r, b = _reference(family, rows, cols)
    assert got.shape == r.shape and torch.isfinite(got).all(), name
    e_p, m_p = _metrics(got, r)
    e_b, m_b = _metrics(b, r)
    print(f"{name}: e_P {e_p:.3e} e_B {e_b:.3e} m_P {m_p:.3e} m_B {m_b:.3e}")
    assert e_p <= F_E * e_b + E_FLOOR and m_p <= F_M * m_b + M_FLOOR and e_p < E_ABS, \
        f"{name}: e_P {e_p:.3e} (torch fp16 {e_b:.3e}), m_P {m_p:.3e} (torch fp16 {m_b:.3e})"


@pytest.mark.parametrize("family", ["sd15", "sdxl"])
@pytest.mark.parametrize("px", [512, 1024])
def test_decode_world1_vs_fp64(family, px):
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    from distrifuser_b200.utils import DistriConfig
    rows = cols = px // 8
    cfg = DistriConfig(height=px, width=px)
    pp = DistriAutoencoderKLPP(_vae(family), cfg)
    z = _latent(rows, cols)
    got = pp.decode(z).sample
    again = pp.decode(z, return_dict=False)[0]
    assert torch.equal(got, again)
    _check(f"{family} {px}^2 world 1", got, family, rows, cols)
    if family == "sd15" and px == 512:                               # another latent size on the same wrapper
        _check("sd15 40x24 latent after 64x64, world 1", pp.decode(_latent(40, 24)).sample, "sd15", 40, 24)


def _gn_check(cfg):
    """DistriGroupNorm(biased_var=True) over this rank's strip of a [1, 64, 7, 4] tensor against nn.GroupNorm of the whole
    tensor: 2 channels per group and 2-3 rows per rank make the local-count Bessel factor 1.04-1.07 and give each strip a
    different mean, so a Bessel or row-weighting error is far above fp16 rounding.  -> (this rank's rows, max |err|)."""
    from distrifuser_b200.modules.pp.groupnorm import DistriGroupNorm
    from distrifuser_b200.utils import PatchParallelismCommManager, row_offset, split_units
    H = 7
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(1, 64, H, 4, generator=g) + torch.arange(H).view(1, 1, H, 1) * 0.7).cuda()
    ref_mod = torch.nn.GroupNorm(32, 64, eps=1e-6)
    with torch.no_grad():
        ref_mod.weight.normal_(1, 0.2, generator=g)
        ref_mod.bias.normal_(0, 0.2, generator=g)
    ref = ref_mod.cuda()(x)
    gn = DistriGroupNorm(copy.deepcopy(ref_mod).half(), cfg)
    gn.biased_var = True
    n, r = cfg.n_device_per_batch, cfg.split_idx()
    units = split_units(H, n)
    gn.row_units = units
    lo = row_offset(units, r)
    strip = x[:, :, lo:lo + units[r]].half().contiguous(memory_format=torch.channels_last)
    cm = PatchParallelismCommManager(cfg)
    gn.set_comm_manager(cm)
    gn(strip)                                                        # registration pass
    cm.create_buffer()
    cm.step_begin(0)
    got = gn(strip).float()
    torch.cuda.synchronize()
    err = (got - ref[:, :, lo:lo + units[r]]).abs().max().item()
    torch.distributed.barrier()                                      # every rank is done with the arenas
    cm.close()
    return units[r], err


def _decode_worker(rank, world, family, shapes, default_cfg, gn_check, port, outdir):
    from torch import distributed as dist
    if torch.cuda.device_count() < world:
        os.environ["DISTRIFUSER_B200_SHARE_GPU"] = "1"
    os.environ["LOCAL_RANK"] = str(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    from distrifuser_b200.models.distri_vae_pp import DistriAutoencoderKLPP
    from distrifuser_b200.utils import DistriConfig
    rows, cols = shapes[0]
    # default_cfg: the pipelines' default config (CFG on, split_batch=True: two patch groups for the UNet); the decoder's
    # world-wide view must override it
    kw = {} if default_cfg else dict(split_batch=False)
    cfg = DistriConfig(height=8 * rows, width=8 * cols, **kw)
    pp = DistriAutoencoderKLPP(_vae(family), cfg)
    imgs = []
    for rows, cols in shapes:                                        # a new shape lays out a new arena
        z = _latent(rows, cols)
        img = pp.decode(z).sample.clone()
        img2 = pp.decode(z).sample                                   # steady state: arena registered, next epoch
        assert torch.equal(img, img2), f"rank {rank}: the second decode differs"
        imgs.append(img.float().cpu())
    gn = _gn_check(pp.view) if gn_check else None
    torch.save((imgs, gn), os.path.join(outdir, f"rank{rank}.pt"))
    torch.cuda.synchronize()
    dist.barrier()
    pp.close()
    dist.destroy_process_group()


def _split(world, family, shapes, default_cfg=False, gn_check=False):
    """-> per rank, (the image of each shape, the GroupNorm check's (rows, max |err|) or None)."""
    from torch import multiprocessing as mp

    from oracle.harness import free_port
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_decode_worker, args=(world, family, shapes, default_cfg, gn_check, free_port(), d), nprocs=world, join=True)
        return [torch.load(os.path.join(d, f"rank{r}.pt")) for r in range(world)]


def _check_split(name, outs, family, shapes):
    for k, (rows, cols) in enumerate(shapes):
        imgs = [o[0][k] for o in outs]
        for r, img in enumerate(imgs):
            assert torch.equal(img, imgs[0]), f"{name}: rank {r} holds another image"
        _check(f"{name}, latent {rows}x{cols}", imgs[0].cuda().half(), family, rows, cols)


@pytest.mark.parametrize("world,rows", [(2, 64), (3, 64)], ids=["n2", "n3-uneven"])
def test_split_decode_share_gpu(world, rows):
    outs = _split(world, "sd15", [(rows, 48)], gn_check=world == 3)
    _check_split(f"sd15 split over {world}", outs, "sd15", [(rows, 48)])
    if world == 3:
        assert [o[1][0] for o in outs] == [3, 2, 2]
        for r, (_, (_, err)) in enumerate(outs):
            assert err < 2e-2, f"rank {r}: DistriGroupNorm(biased_var=True) differs from nn.GroupNorm by {err:.3e}"


def test_split_decode_default_config_and_new_shape():
    """World 2 with the pipelines' default config (CFG split on), then a second latent shape on the same wrapper."""
    shapes = [(64, 48), (40, 24)]
    _check_split("sd15 split over 2, default config", _split(2, "sd15", shapes, default_cfg=True), "sd15", shapes)


def test_split_decode_eight_gpus():
    if torch.cuda.device_count() < 8:
        pytest.skip("needs 8 GPUs")
    _check_split("sdxl 1024^2 split over 8", _split(8, "sdxl", [(128, 128)]), "sdxl", [(128, 128)])


@pytest.mark.parametrize("family", ["sd15", "sdxl"])
def test_from_pretrained_distributed_vae(family):
    """from_pretrained(cfg, distributed_vae=True) through the fake diffusers, whose pipelines end every call that is not
    output_type="latent" with diffusers 0.24's vae.decode(latents / scaling_factor, return_dict=False, generator=generator)."""
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "run_from_pretrained_vae.py"), family], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "OK from_pretrained distributed_vae" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_pipeline_pt_output_is_the_decode_of_its_latents():
    from oracle import workloads as W
    from distrifuser_b200.compat.vae import SD15_VAE, AutoencoderKL
    from distrifuser_b200.pipelines import DistriSDPipeline
    from distrifuser_b200.utils import DistriConfig
    cfg = DistriConfig(height=256, width=192, use_cuda_graph=False)
    torch.manual_seed(3)
    vae = AutoencoderKL(**SD15_VAE)
    pipe = DistriSDPipeline.from_synthetic(cfg, unet_config=W.unet_config("tiny_sd15"), vae=vae)
    run = lambda **kw: pipe(prompt="a photo", num_inference_steps=3, guidance_scale=5.0,
                            generator=torch.Generator().manual_seed(1), **kw).images
    lat = run()
    img = run(output_type="pt")
    with torch.no_grad():
        dec = pipe.pipeline.vae.decode((lat / SD15_VAE["scaling_factor"]).half()).sample
    assert img.shape == (1, 3, 256, 192) and img.min() >= 0 and img.max() <= 1
    assert torch.equal(img, (dec / 2 + 0.5).clamp(0, 1))
    assert torch.equal(run(), lat)                                   # the latent output is unchanged by the decode
