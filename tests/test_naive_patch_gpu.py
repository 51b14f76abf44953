"""GPU tests of the naive patch baseline (parallelism="naive_patch"): the product path (fp16, sm_90a kernels, peer-memory
output gather) against the golden vectors of the unmodified reference NaivePatchUNet (fp32 CPU, gloo), the public pipeline
API against the naive-patch oracle trajectory, and df_output_gather_2d against a torch placement, bit for bit.

Multi-rank cases run on real GPUs when the box has them; otherwise the ranks share cuda:0 through CUDA IPC.  Tolerances are
those of test_unet_gpu.py (helpers.check_parity): mean |err| < 4e-3, max |err| < 4e-2 and PSNR > 45 dB per step."""
import os

import pytest
import torch

from helpers import LoopbackArena, check_parity, psnr
from mp_product import run_product_trajectory, run_product_unet
from oracle.naive_patch import NAIVE_CASES, NaiveCase, run_naive_trajectory

pytestmark = pytest.mark.gpu
CASES = {c.name: c for c in NAIVE_CASES}


def _check(name, outs, gold_path):
    check_parity(name, outs, torch.load(gold_path)["outs"], ranks_identical=True)


@pytest.mark.parametrize("name", ["naive_sdxl_w2_row", "naive_sdxl_w4_col_split", "naive_sdxl_w2_alternate",
                                  "naive_sdxl_w4_alternate", "naive_sd15_w4_col"])
def test_naive_unet_vs_reference(name, golden_dir):
    _check(name, run_product_unet(CASES[name]), os.path.join(golden_dir, f"{name}.pt"))


@pytest.mark.parametrize("name", ["naive_sdxl_w2_alternate", "naive_sdxl_w4_alternate"])
def test_naive_unet_cuda_graph_vs_reference(name, golden_dir):
    """`alternate` with CUDA graphs: steps 0 and 2 replay the row-strip graph, steps 1 and 3 the column-strip graph."""
    _check(name, run_product_unet(CASES[name], use_graph=True), os.path.join(golden_dir, f"{name}.pt"))


@pytest.mark.multigpu(8)
def test_naive_unet_eight_gpus(golden_dir):
    name = "naive_sdxl_w8_split_col"
    _check(name, run_product_unet(CASES[name]), os.path.join(golden_dir, f"{name}.pt"))


@pytest.mark.parametrize("use_graph", [False, True])
def test_naive_world1_is_the_plain_unet(use_graph, golden_dir):
    """At world size 1 naive patch is the wrapped UNet on the whole image: the reference's one-GPU golden applies."""
    case = NaiveCase("w1", world_size=1, scheme="alternate")
    _check("naive w1", run_product_unet(case, use_graph=use_graph), os.path.join(golden_dir, "unet_sdxl_w1.pt"))


@pytest.mark.parametrize("case", [NaiveCase("traj_sdxl_w2_alternate", world_size=2, scheme="alternate"),
                                  NaiveCase("traj_sd15_w2_col", family="tiny_sd15", world_size=2, scheme="col")],
                         ids=lambda c: c.name)
def test_naive_pipeline_trajectory(case):
    """DistriSDXLPipeline / DistriSDPipeline.from_synthetic(DistriConfig(parallelism="naive_patch", ...)) with CUDA graphs,
    8 Euler steps: the final latents are bit-identical on every rank and between two images of one seed (asserted in the
    worker), and within 35 dB of the fp32 naive-patch oracle trajectory."""
    got = run_product_trajectory(case, num_steps=8)
    for lat in got[1:]:
        assert torch.equal(lat, got[0]), "ranks hold different latents"
    want = run_naive_trajectory(case, num_steps=8)
    assert got[0].shape == want.shape
    p = psnr(got[0], want)
    print(f"{case.name}: product vs oracle trajectory {p:.1f} dB")
    assert torch.isfinite(got[0]).all() and p > 35, f"{p:.1f} dB"


# ================================================================================================================ output gather
def _gather_2d(arena, strip, out, B, Cc, H, W, rect):
    from distrifuser_b200 import _lib
    b0, r0, c0, bs, hs, ws = rect
    _lib.check(_lib.lib().df_output_gather_2d(arena.comm, strip.data_ptr(), out.data_ptr(), B, Cc, H, W, bs, hs, ws, b0, r0,
                                              c0, 0, arena.tensor_off[0], torch.cuda.current_stream().cuda_stream),
               "df_output_gather_2d")


def _tiles(B, H, W, rows, cols):
    """(batch0, row0, col0, bs, hs, ws) of every rank: each batch item cut into a grid of row bounds x column bounds."""
    return [(b, rows[i], cols[j], 1, rows[i + 1] - rows[i], cols[j + 1] - cols[j])
            for b in range(B) for i in range(len(rows) - 1) for j in range(len(cols) - 1)]


# rects, index of this rank, whether the 16-byte path applies
GATHER_CASES = {
    "int4-col": (1, 4, 8, 32, _tiles(1, 8, 32, [0, 8], [0, 8, 16, 24, 32]), 2, True),         # SDXL n=8 col shape class
    "half-col": (1, 3, 6, 16, _tiles(1, 6, 16, [0, 6], [0, 4, 8, 12, 16]), 3, False),         # ws = 4
    "half-odd-width": (1, 3, 5, 13, _tiles(1, 5, 13, [0, 5], [0, 4, 7, 10, 13]), 1, False),  # W = 13, ragged ws
    "int4-batch0": (2, 4, 8, 16, _tiles(2, 8, 16, [0, 8], [0, 8, 16]), 3, True),             # CFG split: batch0 = 1
    "half-batch0": (2, 3, 6, 12, _tiles(2, 6, 12, [0, 6], [0, 6, 12]), 3, False),
    "int4-tile": (1, 4, 8, 32, _tiles(1, 8, 32, [0, 4, 8], [0, 16, 32]), 3, True),           # row0 > 0 and col0 > 0
}


@pytest.mark.parametrize("name", list(GATHER_CASES))
def test_output_gather_2d(name):
    """n = 4: the other ranks' strips sit in bank clock[2] (written by the test, flags stamped); this rank scatters its own
    strip at (batch0, row0, col0) and collects the whole image bit-exactly.  The banks of the other epochs are poisoned."""
    B, Cc, H, W, rects, me, vec = GATHER_CASES[name]
    n, E = len(rects), 11
    assert n == 4
    b0, r0, c0, bs, hs, ws = rects[me]
    assert (ws % 8 == 0 and c0 % 8 == 0 and W % 8 == 0 and ws < W) == vec and (c0 > 0 or b0 > 0)
    torch.manual_seed(36)
    img = torch.randn(B, Cc, H, W, device="cuda").half()
    nbytes = img.numel() * 2
    arena = LoopbackArena(n, [nbytes], rank=me)
    try:
        arena.clock[2] = E
        for ep in (E + 1, E - 1):
            arena.slot(ep, 0, 0, nbytes).fill_(float("nan"))
        bank = arena.slot(E, 0, 0, nbytes).view(B, Cc, H, W)
        bank.fill_(float("nan"))
        for r, (rb, rr, rc, rbs, rhs, rws) in enumerate(rects):
            if r != me:
                bank[rb:rb + rbs, :, rr:rr + rhs, rc:rc + rws] = img[rb:rb + rbs, :, rr:rr + rhs, rc:rc + rws]
                arena.flags[0, r] = E
        strip = img[b0:b0 + bs, :, r0:r0 + hs, c0:c0 + ws].contiguous()
        out = torch.full_like(img, float("nan"))
        _gather_2d(arena, strip, out, B, Cc, H, W, rects[me])
        torch.cuda.synchronize()
        assert torch.equal(out, img)
        assert int(arena.flags[0, me].item()) == E
    finally:
        arena.close()


@pytest.mark.parametrize("B,Cc,H,W,me", [(1, 4, 16, 16, 2), (2, 3, 6, 13, 3), (1, 4, 8, 12, 1)])
def test_output_gather_2d_full_width_matches_row_gather(B, Cc, H, W, me):
    """ws == W: the same bytes as df_output_gather, on the same arena state ((1, 4, 8, 12): hs*W = 24, 16-byte path)."""
    from distrifuser_b200 import _lib
    n, E = 4, 5
    per = n // B
    hs = H // per
    rects = [((r // per), (r % per) * hs) for r in range(n)]
    torch.manual_seed(37)
    img = torch.randn(B, Cc, H, W, device="cuda").half()
    nbytes = img.numel() * 2
    outs = []
    for use_2d in (False, True):
        arena = LoopbackArena(n, [nbytes], rank=me)
        try:
            arena.clock[2] = E
            bank = arena.slot(E, 0, 0, nbytes).view(B, Cc, H, W)
            for r, (rb, rr) in enumerate(rects):
                if r != me:
                    bank[rb:rb + 1, :, rr:rr + hs] = img[rb:rb + 1, :, rr:rr + hs]
                    arena.flags[0, r] = E
            b0, r0 = rects[me]
            strip = img[b0:b0 + 1, :, r0:r0 + hs].contiguous()
            out = torch.empty_like(img)
            if use_2d:
                _gather_2d(arena, strip, out, B, Cc, H, W, (b0, r0, 0, 1, hs, W))
            else:
                _lib.check(_lib.lib().df_output_gather(arena.comm, strip.data_ptr(), out.data_ptr(), B, Cc, H, W, 1, hs, b0, r0,
                                                       0, arena.tensor_off[0], torch.cuda.current_stream().cuda_stream),
                           "df_output_gather")
            torch.cuda.synchronize()
            outs.append((out, arena.slot(E, 0, 0, nbytes).clone()))
        finally:
            arena.close()
    assert torch.equal(outs[0][0], img) and torch.equal(outs[1][0], img)
    assert torch.equal(outs[0][1].view(torch.int16), outs[1][1].view(torch.int16))


def test_output_gather_2d_rejects_strips_outside_the_image():
    """Bounds are checked on the host before any launch."""
    from distrifuser_b200 import _lib
    L = _lib.lib()
    c = _lib.null_comm()
    buf = torch.empty(2 * 4 * 8 * 8, dtype=torch.float16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for bs, hs, ws, b0, r0, c0 in [(1, 8, 4, 0, 0, 5), (1, 9, 8, 0, 0, 0), (1, 4, 4, 2, 0, 0), (1, 4, 4, 0, -1, 0)]:
        rc = L.df_output_gather_2d(c, buf.data_ptr(), buf.data_ptr(), 2, 4, 8, 8, bs, hs, ws, b0, r0, c0, 0, 0, st)
        assert rc != 0 and b"df_output_gather_2d" in L.df_last_error()
