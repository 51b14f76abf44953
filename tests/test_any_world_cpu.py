"""Any GPU count up to 8, host side and oracle (CPU): DistriConfig's rank math and groups at world 3, 5, 6 and 7 under a real
process group, the odd-world CFG-split rule, the row rule at patch counts 3, 5, 6 and 7, the arena layout every rank of a
patch group must agree on, and the exactness of the oracle at these counts -- full_sync over 3 strips, with and without the
CFG split, computes the one-device UNet."""
import dataclasses
import os
import tempfile
from types import SimpleNamespace

import pytest
import torch
from torch import distributed as dist
from torch import multiprocessing as mp

from oracle.harness import free_port, run_unet
from oracle.workloads import RaggedCase


def _config_worker(rank, world, port, cfg_on, split, outdir):
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    from distrifuser_b200.utils import DistriConfig, PatchParallelismCommManager
    kw = dict(height=1152, width=1152, do_classifier_free_guidance=cfg_on, split_batch=split, use_cuda_graph=False)
    if cfg_on and split and world % 2:
        with pytest.raises(ValueError, match="split_batch=False"):
            DistriConfig(**kw)
        with pytest.raises(ValueError, match="split_batch=False"):
            DistriConfig(**kw, parallelism="naive_patch")
        open(os.path.join(outdir, f"r{rank}"), "w").close()
        dist.barrier()
        dist.destroy_process_group()
        return
    cfg = DistriConfig(**kw)
    halves = cfg_on and split
    n = world // 2 if halves else world
    assert (cfg.world_size, cfg.rank, cfg.n_device_per_batch) == (world, rank, n)
    assert cfg.batch_idx() == (int(rank >= n) if halves else 0)
    assert cfg.split_idx() == rank % n
    grp = cfg.patch_group_ranks()
    assert grp == list(range(cfg.batch_idx() * n, cfg.batch_idx() * n + n)) and grp[cfg.split_idx()] == rank
    if halves:
        # batch_group: the patch group of this CFG branch; split_group: the two ranks holding the same strip of both branches
        t = torch.tensor([float(rank)])
        dist.all_reduce(t, group=cfg.batch_group)
        assert t.item() == float(sum(grp))
        t = torch.tensor([float(rank)])
        dist.all_reduce(t, group=cfg.split_group)
        assert t.item() == float(2 * cfg.split_idx() + n)
    else:
        assert cfg.batch_group is None and cfg.split_group is None
    # naive patch keeps its whole-strip rule at every patch count: 1152 / 8 = 144 latent rows split over 3 or 6 ranks, and
    # 1024 / 8 = 128 rows do not split over 3, 5, 6 or 7 (nor over 3 per CFG branch at world 6)
    for side in (1152, 1024):
        naive = dict(kw, height=side, width=side, parallelism="naive_patch", split_scheme="alternate")
        if (side // 8) % n == 0:
            assert DistriConfig(**naive).n_device_per_batch == n
        else:
            with pytest.raises(ValueError, match="whole strips"):
                DistriConfig(**naive)
    cm = PatchParallelismCommManager(cfg)
    b = 1 if halves else 2
    cm.register_tensor([2, b, 32, 1, 1, 1], torch.float32, layer_type="gn")
    cm.register_tensor([2, b, 320, 1, 144], torch.float16, layer_type="conv2d")
    cm.register_tensor((b, 144 * 144 // n, 1280), torch.float16, layer_type="attn")
    cm.register_output(2, 4, 144, 144)
    total, bank = cm._layout()
    layout = dict(total=total, bank=bank, off=list(cm.tensor_off), out=cm.output_off, slots=list(cm.slot_bytes))
    assert cm.group_mask() == (1 << n) - 1 and cm.peers_mask() == ((1 << n) - 1) & ~(1 << cfg.split_idx())
    gathered = [None] * world
    dist.all_gather_object(gathered, (cfg.batch_idx(), layout))
    assert all(lay == layout for bi, lay in gathered if bi == cfg.batch_idx()), "ranks of one patch group disagree"
    open(os.path.join(outdir, f"r{rank}"), "w").close()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [3, 5, 6, 7])
@pytest.mark.parametrize("cfg_on,split", [(True, True), (True, False), (False, True)], ids=["cfg-split", "cfg-nosplit", "nocfg"])
def test_config_rank_math_any_world(world, cfg_on, split):
    """n_device_per_batch, batch_idx, split_idx, patch_group_ranks, the batch / split groups and the arena layout; an odd world
    with the CFG split raises ValueError naming split_batch=False."""
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_config_worker, args=(world, free_port(), cfg_on, split, d), nprocs=world, join=True)
        assert len(os.listdir(d)) == world


def test_power_of_two_check_kept():
    from distrifuser_b200.utils import is_power_of_2
    assert [w for w in range(1, 9) if is_power_of_2(w)] == [1, 2, 4, 8]


@pytest.mark.parametrize("n", [3, 5, 6, 7])
@pytest.mark.parametrize("u", [4, 8], ids=["sdxl", "sd15"])
def test_rows_at_every_level_any_n(n, u):
    """split_units / patch_rows / row_offset at every UNet level for every unit count from n to 64: rank r holds units_r * u
    / 2^l rows at level l, starting at the prefix sum, and every rank finds all of them from its own h."""
    from distrifuser_b200.utils import patch_rows, row_offset, split_units
    for U in range(n, 65):
        units = split_units(U, n)
        assert len(units) == n and sum(units) == U and units == sorted(units, reverse=True)
        assert units == [U // n + 1] * (U % n) + [U // n] * (n - U % n)
        level = 0
        while u >> level >= 1:
            want = [k * (u >> level) for k in units]
            assert sum(want) == U * u >> level
            for r in range(n):
                rows = patch_rows(units, r, want[r])
                assert rows == want and row_offset(rows, r) == sum(want[:r])
                assert row_offset(rows, r) + rows[r] == (row_offset(rows, r + 1) if r + 1 < n else U * u >> level)
            level += 1


def test_sdxl_row_plans():
    """SDXL 1024^2 (32 units of 4 latent rows): 11 / 11 / 10 units at n = 3, 6 / 6 / 5 / 5 / 5 / 5 at n = 6; 1536^2 (48
    units) splits evenly at every n in {1, 2, 3, 4, 6, 8}."""
    from distrifuser_b200.models.distri_sdxl_unet_pp import row_plan
    sdxl = SimpleNamespace(config=SimpleNamespace(block_out_channels=[320, 640, 1280]))     # two downsamplers: u = 4
    plan = lambda h, n: row_plan(sdxl, SimpleNamespace(height=h, n_device_per_batch=n))
    assert plan(1024, 3) == [11, 11, 10]
    assert plan(1024, 6) == [6, 6, 5, 5, 5, 5]
    assert plan(1024, 5) == [7, 7, 6, 6, 6] and plan(1024, 7) == [5, 5, 5, 5, 4, 4, 4]
    for n in (1, 2, 3, 4, 6, 8):
        assert plan(1536, n) == [48 // n] * n


def _plan_worker(rank, world, port, split, lat_h, want, outdir):
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    from oracle import workloads as W
    from distrifuser_b200.compat.unet_2d_condition import UNet2DConditionModel
    from distrifuser_b200.models.distri_sdxl_unet_pp import DistriUNetPP
    from distrifuser_b200.utils import DistriConfig, PatchParallelismCommManager, patch_rows
    cfg = DistriConfig(height=8 * lat_h, width=224, split_batch=split, use_cuda_graph=False)
    unet = DistriUNetPP(UNet2DConditionModel(**W.unet_config("tiny_sdxl")), cfg)
    assert unet.row_units == want, f"rank {rank}: row plan {unet.row_units}"
    r = cfg.split_idx()
    # what the wrappers register at each level of the tiny SDXL (width 28 latent columns): GroupNorm statistics, conv halo rows
    # and self-attention K/V slots at the LARGEST strip's size
    cm = PatchParallelismCommManager(cfg)
    b, w = (1 if split else 2), 28
    for level, C in enumerate((64, 128, 256)):
        h = unet.row_units[r] * 4 >> level
        cm.register_tensor([2, b, 32, 1, 1, 1], torch.float32, layer_type="gn")
        cm.register_tensor([2, b, C, 1, w >> level], torch.float16, layer_type="conv2d")
        lens = patch_rows(unet.row_units, r, h * (w >> level))
        cm.register_tensor((b, h * (w >> level), 2 * C), torch.float16, layer_type="attn", slot_bytes=b * max(lens) * 2 * C * 2)
    cm.register_output(2, 4, lat_h, 28)
    total, bank = cm._layout()
    layout = dict(total=total, bank=bank, off=list(cm.tensor_off), out=cm.output_off, slots=list(cm.slot_bytes))
    gathered = [None] * world
    dist.all_gather_object(gathered, layout)
    assert all(lay == layout for lay in gathered), "ranks disagree on the arena layout"
    open(os.path.join(outdir, f"r{rank}"), "w").close()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,split,lat_h,units", [(3, False, 40, [4, 3, 3]), (6, False, 36, [2, 2, 2, 1, 1, 1]),
                                                     (6, True, 40, [4, 3, 3])], ids=["n3", "n6", "w6-split-n3"])
def test_row_plan_and_arena_layout_any_n(world, split, lat_h, units):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_plan_worker, args=(world, free_port(), split, lat_h, units, d), nprocs=world, join=True)
        assert len(os.listdir(d)) == world


EXACT = [
    (RaggedCase("sdxl_n3", world_size=3, mode="full_sync", steps=2, lat_h=40), [4, 3, 3]),
    (RaggedCase("sdxl_w6_split_n3", world_size=6, split_batch=True, mode="full_sync", steps=2, lat_h=40), [4, 3, 3]),
]


@pytest.mark.parametrize("case,units", EXACT, ids=[c.name for c, _ in EXACT])
def test_full_sync_any_world_equals_one_device(case, units):
    """Without the local-count Bessel factor, full_sync over 3 strips (one patch group, or one per CFG branch at world 6) is
    the whole-image UNet (fp32, within 1e-5)."""
    got = run_unet(case, bessel=False, row_units=units)
    want = run_unet(dataclasses.replace(case, world_size=1), bessel=False)
    for t, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape == (2, 4, case.lat_h, case.lat_w)
        err = (a - b).abs().max().item()
        assert err < 1e-5, f"step {t}: max |err| {err:.2e}"
