"""CPU checks of the naive patch baseline (parallelism="naive_patch"): the fp32 oracle against the golden vectors of the
unmodified reference NaivePatchUNet, the DistriConfig rules for naive patch, and the premise the method rests on -- over a
denoising trajectory, displaced patch parallelism stays close to the one-device result while naive splitting does not."""
import os
import tempfile

import pytest
import torch
from torch import distributed as dist
from torch import multiprocessing as mp

from helpers import psnr
from oracle import harness, workloads
from oracle.naive_patch import NAIVE_CASES, NaiveCase, run_naive_trajectory, run_naive_unet


@pytest.mark.parametrize("case", NAIVE_CASES, ids=lambda c: c.name)
def test_naive_oracle_matches_reference(case, golden_dir):
    gold = torch.load(os.path.join(golden_dir, f"{case.name}.pt"))
    assert gold["case"] == case.__dict__
    outs = run_naive_unet(case, impl="oracle")
    assert len(outs) == len(gold["outs"]) == case.steps
    for t, (a, b) in enumerate(zip(outs, gold["outs"])):
        assert a.shape == b.shape == (case.batch, 4, case.latent, case.latent)
        err = (a - b).abs().max().item()
        assert err < 1e-4, f"{case.name} step {t}: max |oracle - reference| {err:.2e}"


def test_naive_patch_config_world1():
    from distrifuser_b200.utils import DistriConfig
    for scheme in ("row", "col", "alternate"):
        cfg = DistriConfig(height=256, width=256, parallelism="naive_patch", split_scheme=scheme)
        assert (cfg.parallelism, cfg.split_scheme, cfg.n_device_per_batch, cfg.split_idx()) == ("naive_patch", scheme, 1, 0)
    for scheme in ("diagonal", "rows", None):
        with pytest.raises(NotImplementedError):
            DistriConfig(height=256, width=256, parallelism="naive_patch", split_scheme=scheme)
    with pytest.raises(NotImplementedError):
        DistriConfig(parallelism="tensor", split_scheme="row")
    # the reference ignores split_scheme under patch parallelism, and so does this package
    for scheme in ("col", "alternate", "anything"):
        assert DistriConfig(height=256, width=256, parallelism="patch", split_scheme=scheme).split_scheme == scheme


def _config_worker(rank, world, port, outdir):
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method=f"tcp://127.0.0.1:{port}")
    from distrifuser_b200.utils import DistriConfig
    # world 4 without a CFG split: 4 strips per image; with it: 2 strips per CFG half
    ok = [(256, 256, False, s) for s in ("row", "col", "alternate")] + [(8 * 30, 256, False, "col"),
                                                                          (256, 8 * 30, False, "row"),
                                                                          (8 * 30, 8 * 30, True, "alternate")]
    bad = [(8 * 30, 256, False, "row"), (256, 8 * 30, False, "col"), (8 * 30, 256, False, "alternate"),
           (256, 8 * 30, False, "alternate"), (8 * 33, 8 * 33, True, "row"), (8 * 33, 8 * 33, True, "col")]
    for h, w, split, scheme in ok:
        cfg = DistriConfig(height=h, width=w, split_batch=split, parallelism="naive_patch", split_scheme=scheme)
        assert cfg.n_device_per_batch == (world // 2 if split else world)
        assert cfg.split_idx() == rank % cfg.n_device_per_batch and cfg.batch_idx() == (int(rank >= world // 2) if split else 0)
    for h, w, split, scheme in bad:
        with pytest.raises(ValueError, match="whole strips"):
            DistriConfig(height=h, width=w, split_batch=split, parallelism="naive_patch", split_scheme=scheme)
    open(os.path.join(outdir, f"r{rank}"), "w").close()
    dist.barrier()
    dist.destroy_process_group()


def test_naive_patch_config_whole_strips():
    """At world 4 a strip must be a whole number of latent rows (row), columns (col) or both (alternate)."""
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_config_worker, args=(4, harness.free_port(), d), nprocs=4, join=True)
        assert len(os.listdir(d)) == 4


def test_naive_patch_premise_on_trajectories():
    """Tiny SDXL, latent 32, 8 Euler steps, guidance 5: final latents against the one-device trajectory.  Naive patch at
    n=2 (every scheme) stays under 40 dB; DistriFusion (displaced patch parallelism, one warm-up step) stays over 50 dB.
    Whole trajectories are compared: each call of the parity workloads draws fresh inputs, so a single call scores a
    1-step-stale method on data it never saw."""
    steps = 8
    full = run_naive_trajectory(NaiveCase("one_device", world_size=1), num_steps=steps)
    naive = {s: psnr(run_naive_trajectory(NaiveCase(f"n2_{s}", world_size=2, scheme=s), num_steps=steps), full, floor=1e-30)
             for s in ("row", "col", "alternate")}
    distri = psnr(harness.run_trajectory(workloads.UNetCase("pp_n2", world_size=2, split_batch=False, warmup_steps=1),
                                         num_steps=steps), full, floor=1e-30)
    print(f"PSNR vs one device: naive n=2 {naive}, DistriFusion n=2 {distri:.1f} dB")
    assert all(p < 40 for p in naive.values()), naive
    assert distri > 50, distri
