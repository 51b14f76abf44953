"""ControlNet without a GPU: the compat model against the diffusers-0.24 restatement, the zero-weight premise, the oracle's
patch-parallel UNet + ControlNet against one device, and the host-side checks of the patch-parallel wrapper."""
from dataclasses import replace
from types import SimpleNamespace

import pytest
import torch

from helpers import psnr
from oracle import workloads as W
from oracle.harness import run_unet

TINY = ("tiny_sdxl", "tiny_sd15")


@pytest.fixture(autouse=True)
def _plain_attention(monkeypatch):
    """The compat Attention only runs inside the GPU wrappers; on the CPU it is plain SDPA, as in test_compat_unet.py."""
    from distrifuser_b200.compat import unet_2d_condition as compat
    from test_compat_unet import _sdpa_forward
    monkeypatch.setattr(compat.Attention, "forward", _sdpa_forward)


def _compat_pair(family, zero=False):
    from distrifuser_b200.compat.controlnet import ControlNetModel
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    ucfg = W.unet_config(family)
    stub_unet, stub_cn = W.make_unet(family, 0), W.make_controlnet(family, 0, zero=zero)
    unet, cn = UNet2DConditionModel(**ucfg).eval(), ControlNetModel(**ucfg).eval()
    unet.load_state_dict(stub_unet.state_dict(), strict=True)
    cn.load_state_dict(stub_cn.state_dict(), strict=True)
    return ucfg, stub_unet, stub_cn, unet, cn


def _inputs(family, ucfg, lat=16):
    case = W.UNetCase("cn", family=family, latent=lat)
    inp = W.unet_inputs(case, 0, ucfg)
    return inp, W.cond_image(case).expand(case.batch, -1, -1, -1)


@pytest.mark.parametrize("family", TINY)
def test_compat_controlnet_matches_restatement(family):
    ucfg, stub_unet, stub_cn, unet, cn = _compat_pair(family)
    inp, cond = _inputs(family, ucfg)
    n_res = {"tiny_sdxl": 9, "tiny_sd15": 12}[family]
    with torch.no_grad():
        d_ref, m_ref = stub_cn(inp["sample"], inp["timestep"], inp["encoder_hidden_states"], cond, 0.7,
                               added_cond_kwargs=inp["added_cond_kwargs"])
        d, m = cn(inp["sample"], inp["timestep"], inp["encoder_hidden_states"], cond, 0.7,
                  added_cond_kwargs=inp["added_cond_kwargs"])
        assert len(d) == len(d_ref) == n_res
        for a, b in zip([*d, m], [*d_ref, m_ref]):
            assert b.abs().max() > 1e-3                                   # the drawn zero convs give non-zero residuals
            torch.testing.assert_close(a, b, rtol=0, atol=1e-5)
        want = stub_unet(inp["sample"], inp["timestep"], inp["encoder_hidden_states"],
                         added_cond_kwargs=inp["added_cond_kwargs"], down_block_additional_residuals=d_ref,
                         mid_block_additional_residual=m_ref, return_dict=False)[0]
        got = unet(inp["sample"], inp["timestep"], inp["encoder_hidden_states"], added_cond_kwargs=inp["added_cond_kwargs"],
                   down_block_additional_residuals=d, mid_block_additional_residual=m, return_dict=False)[0]
    torch.testing.assert_close(got, want, rtol=0, atol=1e-5)


@pytest.mark.parametrize("family", TINY)
def test_from_unet_copies_encoder_and_loads_strict(family):
    from distrifuser_b200.compat.controlnet import ControlNetModel
    _, stub_unet, stub_cn, unet, _ = _compat_pair(family)
    cn = ControlNetModel.from_unet(unet)
    sd = cn.state_dict()
    for k, v in unet.state_dict().items():
        if k.split(".")[0] in ("conv_in", "time_embedding", "add_embedding", "down_blocks", "mid_block"):
            assert torch.equal(sd[k], v), k
    assert set(sd) == set(stub_cn.state_dict())
    cn.load_state_dict(stub_cn.state_dict(), strict=True)
    assert torch.equal(cn.controlnet_mid_block.weight, stub_cn.controlnet_mid_block.weight)


@pytest.mark.parametrize("family", TINY)
def test_fresh_controlnet_leaves_unet_output_unchanged(family):
    from distrifuser_b200.compat.controlnet import ControlNetModel
    _, _, _, unet, _ = _compat_pair(family)
    cn = ControlNetModel.from_unet(unet).eval()
    for z in [cn.controlnet_cond_embedding.conv_out, *cn.controlnet_down_blocks, cn.controlnet_mid_block]:
        assert not any(p.any() for p in z.parameters())
    inp, cond = _inputs(family, W.unet_config(family))
    with torch.no_grad():
        d, m = cn(inp["sample"], inp["timestep"], inp["encoder_hidden_states"], cond, 1.0,
                  added_cond_kwargs=inp["added_cond_kwargs"])
        kw = dict(added_cond_kwargs=inp["added_cond_kwargs"], return_dict=False)
        a = unet(inp["sample"], inp["timestep"], inp["encoder_hidden_states"], down_block_additional_residuals=d,
                 mid_block_additional_residual=m, **kw)[0]
        b = unet(inp["sample"], inp["timestep"], inp["encoder_hidden_states"], **kw)[0]
    assert torch.equal(a, b)


FULL_SYNC_CASES = (
    W.UNetCase("cn_sdxl_w2_nosplit", world_size=2, split_batch=False, mode="full_sync", steps=2),
    W.UNetCase("cn_sdxl_w4_split", world_size=4, mode="full_sync", steps=2),
    W.UNetCase("cn_sdxl_w4_nosplit", world_size=4, split_batch=False, mode="full_sync", steps=2),
    W.RaggedCase("cn_sdxl_w3_ragged", world_size=3, mode="full_sync", steps=2),
    W.UNetCase("cn_sd15_w2_nosplit", family="tiny_sd15", world_size=2, split_batch=False, mode="full_sync", steps=2),
)


@pytest.mark.parametrize("case", FULL_SYNC_CASES, ids=lambda c: c.name)
def test_oracle_full_sync_equals_one_device(case):
    """Every exchange synchronous: the patch-parallel UNet + ControlNet is the one-device forward (uneven strips: without the
    local-count Bessel factor, which differs between strip heights)."""
    got = run_unet(case, bessel=False, controlnet="drawn")
    want = run_unet(replace(case, world_size=1), controlnet="drawn")
    for a, b in zip(got, want):
        torch.testing.assert_close(a, b, rtol=0, atol=1e-5)


# Measured on the CPU oracle (seeded tiny SDXL, world 2, warmup 1): 75.0 / 74.4 / 21.4 / 23.0 dB at steps 0-3.  Steps 0 and 1 are
# synchronous and differ from one device only by the local-count Bessel factor; from step 2 on, the inputs of these synthetic
# workloads are independent draws per step, so one-step-stale activations are far from the fresh ones.  The bar records that
# level, ~3 dB under the lowest.
ASYNC_PSNR_DB = 18.0


def test_oracle_corrected_async_gn_psnr():
    case = W.UNetCase("cn_sdxl_w2_async", world_size=2, split_batch=False, mode="corrected_async_gn", steps=4)
    got, want = run_unet(case, controlnet="drawn"), run_unet(replace(case, world_size=1), controlnet="drawn")
    ps = [psnr(a, b) for a, b in zip(got, want)]
    print("corrected_async_gn PSNR per step:", [f"{p:.1f}" for p in ps])
    assert min(ps) > ASYNC_PSNR_DB, ps


# ---------------------------------------------------------------------------------------------------------------- host logic
def test_pixel_row_plan_is_eight_times_latent_plan():
    from distrifuser_b200.compat.controlnet import ControlNetModel
    from distrifuser_b200.models.distri_sdxl_unet_pp import row_plan
    from distrifuser_b200.utils import patch_rows
    cn = ControlNetModel(**W.unet_config("tiny_sdxl"))
    for n, height in ((3, 8 * 36), (2, 8 * 32), (5, 1024), (7, 1216)):
        units = row_plan(cn, SimpleNamespace(n_device_per_batch=n, height=height))
        for r in range(n):
            lat = height // 8 * units[r] // sum(units)
            assert patch_rows(units, r, 8 * lat) == [8 * x for x in patch_rows(units, r, lat)]
            assert sum(patch_rows(units, r, 8 * lat)) == height


def _cpu_wrapper(parallelism="patch"):
    from distrifuser_b200.compat.controlnet import ControlNetModel
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.pipelines import _wrap
    from distrifuser_b200.utils import DistriConfig
    ucfg = W.unet_config("tiny_sdxl")
    cfg = DistriConfig(height=128, width=128, parallelism=parallelism, use_cuda_graph=False)
    return _wrap(UNet2DConditionModel(**ucfg).eval(), cfg, ControlNetModel(**ucfg).eval()), ucfg


def test_bad_conditioning_image_and_outside_residuals_raise():
    model, ucfg = _cpu_wrapper()
    inp = W.unet_inputs(W.UNetCase("cn", latent=16), 0, ucfg)
    with pytest.raises(ValueError, match="pixel resolution"):
        model(**inp, controlnet_cond=torch.zeros(2, 3, 64, 128))
    with pytest.raises(ValueError, match="controlnet_cond"):
        model(**inp)
    with pytest.raises(ValueError, match="residuals from outside"):
        model(**inp, down_block_additional_residuals=[torch.zeros(1)], controlnet_cond=torch.zeros(2, 3, 128, 128))


def test_naive_patch_with_controlnet_raises():
    with pytest.raises(NotImplementedError, match="patch parallelism only"):
        _cpu_wrapper("naive_patch")

