"""Patch parallelism on uneven row strips, host side and oracle (CPU): the row rule, the ValueError of heights that cannot be
split, the arena layout every rank of a patch group must agree on, and the exactness of the uneven oracle -- full_sync over
uneven strips computes the one-device UNet."""
import os
import tempfile

import pytest
import torch
from torch import distributed as dist
from torch import multiprocessing as mp

from oracle.harness import free_port, run_unet
from oracle.workloads import RaggedCase


def test_split_units_rule():
    from distrifuser_b200.utils import split_units
    assert split_units(9, 4) == [3, 2, 2, 2]
    assert split_units(9, 2) == [5, 4]
    assert split_units(5, 4) == [2, 1, 1, 1]
    for U in range(1, 40):
        for n in (1, 2, 4, 8):
            if U < n:
                continue
            units = split_units(U, n)
            assert sum(units) == U and max(units) - min(units) <= 1 and units == sorted(units, reverse=True)
            if U % n == 0:
                assert units == [U // n] * n


@pytest.mark.parametrize("U,n,u", [(9, 4, 4), (9, 2, 4), (5, 4, 8), (32, 4, 4), (16, 8, 8), (7, 2, 4)])
def test_rows_at_every_level_and_prefix_sums(U, n, u):
    """Rank r holds units_r * u / 2^l rows at level l, starting at the prefix sum; any rank finds all of them from its own h."""
    from distrifuser_b200.utils import patch_rows, row_offset, split_units
    units = split_units(U, n)
    S = U * u
    level = 0
    while u >> level >= 1:
        want = [k * (u >> level) for k in units]
        assert sum(want) == S >> level
        for r in range(n):
            rows = patch_rows(units, r, want[r])
            assert rows == want
            assert row_offset(rows, r) == sum(want[:r])
            if U % n == 0:
                assert rows == [(S >> level) // n] * n and row_offset(rows, r) == r * ((S >> level) // n)
        level += 1
    with pytest.raises(ValueError):
        patch_rows([3, 2], 1, 3)                      # 3 rows of a 2-unit strip: not whole rows per unit


def _plan_worker(rank, world, port, outdir):
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    from oracle import workloads as W
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.models.distri_sdxl_unet_pp import DistriUNetPP
    from distrifuser_b200.utils import DistriConfig, PatchParallelismCommManager, patch_rows
    ucfg = W.unet_config("tiny_sdxl")
    for S in (34, 12):                                # 34 % 4 != 0; 12 rows = 3 units < 4 ranks
        cfg = DistriConfig(height=8 * S, width=224, split_batch=False, use_cuda_graph=False)
        try:
            DistriUNetPP(UNet2DConditionModel(**ucfg), cfg)
            raise AssertionError(f"latent height {S} over 4 ranks was accepted")
        except ValueError as e:
            assert ("multiple of 4" in str(e)) if S == 34 else ("at least 4 units" in str(e)), str(e)
    cfg = DistriConfig(height=8 * 36, width=224, split_batch=False, use_cuda_graph=False)
    unet = DistriUNetPP(UNet2DConditionModel(**ucfg), cfg)
    assert unet.row_units == [3, 2, 2, 2]
    r = cfg.split_idx()
    # what the wrappers register at each level of the tiny SDXL (b = 2, width 28 latent columns): GroupNorm statistics, conv
    # halo rows of their own shape, and self-attention K/V slots at the LARGEST strip's size
    cm = PatchParallelismCommManager(cfg)
    b, w = 2, 28
    for level, C in enumerate((64, 128, 256)):
        h = unet.row_units[r] * 4 >> level
        cm.register_tensor([2, b, 32, 1, 1, 1], torch.float32, layer_type="gn")
        cm.register_tensor([2, b, C, 1, w >> level], torch.float16, layer_type="conv2d")
        lens = patch_rows(unet.row_units, r, h * (w >> level))
        cm.register_tensor((b, h * (w >> level), 2 * C), torch.float16, layer_type="attn", slot_bytes=b * max(lens) * 2 * C * 2)
    cm.register_output(2, 4, 36, 28)
    total, bank = cm._layout()
    layout = dict(total=total, bank=bank, off=list(cm.tensor_off), out=cm.output_off, slots=list(cm.slot_bytes))
    gathered = [None] * world
    dist.all_gather_object(gathered, layout)
    assert all(lay == layout for lay in gathered), "ranks of one patch group disagree on the arena layout"
    torch.save(layout, os.path.join(outdir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_row_plan_and_arena_layout_multirank():
    """world 4, no CFG split: n = 4 ranks over a 36-row latent (9 units of 4 rows): [3, 2, 2, 2] units, one arena layout."""
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_plan_worker, args=(4, free_port(), d), nprocs=4, join=True)
        assert len(os.listdir(d)) == 4


EXACT = [
    (RaggedCase("sdxl_n2", world_size=2, mode="full_sync", steps=2), [5, 4]),
    (RaggedCase("sdxl_n4", world_size=4, mode="full_sync", steps=2), [3, 2, 2, 2]),
    (RaggedCase("sd15_n4", family="tiny_sd15", world_size=4, mode="full_sync", steps=2, lat_h=40, lat_w=24), [2, 1, 1, 1]),
]


@pytest.mark.parametrize("case,units", EXACT, ids=[c.name for c, _ in EXACT])
def test_uneven_full_sync_equals_one_device(case, units):
    """Without the local-count Bessel factor, full_sync over uneven strips is the whole-image UNet (fp32, within 1e-5)."""
    import dataclasses
    got = run_unet(case, bessel=False, row_units=units)
    want = run_unet(dataclasses.replace(case, world_size=1), bessel=False)
    for t, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape == (2, 4, case.lat_h, case.lat_w)
        err = (a - b).abs().max().item()
        assert err < 1e-5, f"step {t}: max |err| {err:.2e}"


@pytest.mark.parametrize("world,units", [(2, [5, 4]), (4, [3, 2, 2, 2])])
def test_uneven_corrected_warmup_equals_full_sync(world, units):
    """With the Bessel factor, the synchronous warm-up steps of corrected_async_gn compute what full_sync computes."""
    sync = run_unet(RaggedCase("full", world_size=world, mode="full_sync", warmup_steps=2, steps=3), row_units=units)
    corr = run_unet(RaggedCase("corr", world_size=world, mode="corrected_async_gn", warmup_steps=2, steps=3), row_units=units)
    for t, (a, b) in enumerate(zip(corr, sync)):
        err = (a - b).abs().max().item()
        assert err < 1e-5, f"warm-up step {t}: max |err| {err:.2e}"
