"""ControlNet on the H100: the one-launch zero-conv kernel against fp32 torch, and the patch-parallel UNet + ControlNet product
(mp_product.py) against the fp32 oracle (oracle/harness.py), eager and with CUDA graphs.  With fewer GPUs than ranks the ranks
share cuda:0, as in mp_product.py."""
import dataclasses

import pytest
import torch

import mp_product as MP
from helpers import check_parity, psnr
from oracle import workloads as W
from oracle.harness import run_trajectory, run_unet

pytestmark = pytest.mark.gpu

# (C, tokens) of every zero conv of one call.  SDXL 1024^2 (latent 128) on the rank with 10 of 32 row units at n = 3: strip
# tokens 40*128, 20*64, 10*32; SD1.x 768^2 (latent 96) on the rank with 4 of 12 units at n = 5 (8-row units): 32*96 ... 4*12.
# Several token counts are not multiples of the 128-row tile.
SDXL_CONVS = [(320, 5120)] * 4 + [(640, 1280)] * 3 + [(1280, 320)] * 2 + [(1280, 320)]
SD15_CONVS = ([(320, 3072)] * 4 + [(640, 768)] * 3 + [(1280, 192)] * 3 + [(1280, 48)] * 2 + [(1280, 48)])
ODD_CONVS = [(320, 1000), (640, 250), (1280, 63)]
TINY_SD15_CONVS = [(80, 1000), (160, 250), (320, 63)]          # widths that are not multiples of the 64-wide K block


def _problems(spec, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs, convs = [], []
    for c, m in spec:
        xs.append(torch.randn(1, c, 1, m, device="cuda", generator=g).half().contiguous(memory_format=torch.channels_last))
        conv = torch.nn.Conv2d(c, c, 1).cuda().half()
        with torch.no_grad():
            conv.weight.copy_(torch.randn(conv.weight.shape, device="cuda", generator=g) / c ** 0.5)
            conv.bias.copy_(torch.randn(conv.bias.shape, device="cuda", generator=g) * 0.1)
        convs.append(conv)
    return xs, convs


def _ref(xs, convs, s):
    return [(torch.nn.functional.conv2d(x.float(), cv.weight.float(), cv.bias.float()).half().float() * s) for x, cv in zip(xs, convs)]


@pytest.mark.parametrize("spec", [SDXL_CONVS, SD15_CONVS, ODD_CONVS, TINY_SD15_CONVS, SDXL_CONVS[:1], [(1280, 63)]],
                         ids=["sdxl10", "sd15_13", "odd_tokens", "k_tail", "one_sdxl", "one_odd"])
def test_zero_convs_match_fp32(spec):
    from distrifuser_b200 import ops
    xs, convs = _problems(spec)
    scale = torch.tensor([0.75], device="cuda")
    outs = ops.controlnet_zero_convs(xs, convs, scale)
    torch.cuda.synchronize()
    for o, r in zip(outs, _ref(xs, convs, 0.75)):
        assert o.shape == r.shape
        err = (o.float() - r).abs()
        assert (err <= 4e-3 + 2e-3 * r.abs()).all(), f"max err {err.max():.3e}"


def test_zero_convs_graph_replay_reads_device_scale():
    from distrifuser_b200 import ops
    xs, convs = _problems(SDXL_CONVS, seed=1)
    scale = torch.tensor([1.0], device="cuda")
    ops.controlnet_zero_convs(xs, convs, scale)                    # first launch outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = ops.controlnet_zero_convs(xs, convs, scale)
    got = {}
    for s in (1.0, 0.25, -0.5):
        scale.fill_(s)
        g.replay()
        torch.cuda.synchronize()
        got[s] = [o.float().clone() for o in outs]
        for o, r in zip(got[s], _ref(xs, convs, s)):
            assert ((o - r).abs() <= 4e-3 + 2e-3 * r.abs()).all()
    assert not torch.equal(got[1.0][0], got[0.25][0])


def test_zero_convs_reject_bad_shapes():
    from distrifuser_b200 import ops
    xs, convs = _problems([(320, 128)])
    scale = torch.ones(1, device="cuda")
    bad_n = torch.nn.Conv2d(320, 12, 1).cuda().half()              # N % 8 != 0
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.controlnet_zero_convs(xs, [bad_n], scale)
    x100 = torch.randn(1, 100, 1, 128, device="cuda").half().contiguous(memory_format=torch.channels_last)
    with pytest.raises(RuntimeError, match="unsupported shape"):    # K % 8 != 0
        ops.controlnet_zero_convs([x100], [torch.nn.Conv2d(100, 80, 1).cuda().half()], scale)
    with pytest.raises(RuntimeError, match="problems"):             # longer list than one launch takes
        ops.controlnet_zero_convs(xs * 14, convs * 14, scale)


# ------------------------------------------------------------------------------------------------ UNet + ControlNet vs oracle
CASES = (
    W.UNetCase("cn_sdxl_w1", world_size=1, steps=3),
    W.UNetCase("cn_sdxl_w2_nosplit", world_size=2, split_batch=False, steps=3),
    W.UNetCase("cn_sdxl_w4_split", world_size=4, steps=3),
    W.RaggedCase("cn_sdxl_w3_ragged", world_size=3, steps=3),
    W.UNetCase("cn_sd15_w2_nosplit", family="tiny_sd15", world_size=2, split_batch=False, mode="stale_gn", steps=3),
)


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_unet_controlnet_vs_oracle(case, use_graph):
    want = run_unet(case, controlnet="drawn")
    got = MP.run_product_unet(case, use_graph=use_graph, controlnet="drawn")
    check_parity(case.name, got, want, ranks_identical=True)


def test_zero_controlnet_output_bit_identical():
    """A zero-initialised ControlNet adds exact zeros: the product output equals the same pipeline without a ControlNet."""
    case = W.UNetCase("cn_sdxl_w2_zero", world_size=2, split_batch=False, steps=3)
    for r, (without, with_cn) in enumerate(MP.run_zero_premise(case)):
        for t, (x, y) in enumerate(zip(without, with_cn)):
            assert torch.equal(x, y), f"rank {r} step {t}: max |diff| {(x - y).abs().max():.3e}"


def test_graph_replay_honours_new_scale():
    """One captured graph, a different conditioning scale per step: each step matches the oracle at that scale."""
    case = W.UNetCase("cn_sdxl_w1_scale", world_size=1, steps=3)
    scales = [1.0, 0.5, 0.0]
    got = MP.run_product_unet(case, use_graph=True, controlnet="drawn", scale=scales)
    for t, s in enumerate(scales):
        want = run_unet(dataclasses.replace(case, steps=t + 1), controlnet="drawn", scale=s)[t]
        check_parity(f"{case.name} scale {s}", [[got[0][t]]], [want])


def test_pipeline_trajectory_with_controlnet():
    case = W.UNetCase("cn_sdxl_w2_traj", world_size=2, split_batch=False, warmup_steps=2)
    got = MP.run_product_trajectory(case, controlnet="drawn")
    for r in range(1, len(got)):
        assert torch.equal(got[r], got[0]), f"rank {r} final latents differ from rank 0"
    want = run_trajectory(case, controlnet="drawn")
    p = psnr(got[0], want)
    assert p > 35, f"trajectory PSNR {p:.1f} dB"


def test_full_size_sdxl_unet_controlnet_step_vs_oracle():
    """The full SDXL UNet and a full-size ControlNet (random init, drawn zero convs), 512x512, one CFG step, world 1, against the
    fp32 oracle; the bar of test_full_size_sdxl_unet_step_vs_oracle."""
    case = dataclasses.replace(W.UNetCase("cn_sdxl_full_512", family="sdxl", world_size=1, latent=64), steps=1)
    got = MP.run_product_unet(case, controlnet="drawn")[0][0]
    want = run_unet(case, controlnet="drawn")[0]
    assert got.shape == want.shape == (2, 4, 64, 64)
    err = (got - want).abs()
    std = want.std().item()
    p = psnr(got, want)
    assert torch.isfinite(got).all()
    assert err.mean().item() < 1.2e-2 * std and err.max().item() < 0.12 * std and p > 45, \
        f"mean {err.mean():.2e} max {err.max():.2e} std {std:.3f} psnr {p:.1f} dB"
