"""GPU tests of patch parallelism and the naive patch baseline at GPU counts that are not powers of two.

Kernels, at patch counts 3, 5 and 7 with this rank first, in the middle and last: attention over that many K/V segments of
unequal length against an fp32 SDPA, the rows-weighted GroupNorm statistics (plain and with the fused halo) against torch,
the halo push / assemble and the activation publication over communicators whose members have DISTINCT arenas (so that a wrong
neighbour or mask bit lands in the wrong member's memory), and the output gather of 3 / 5 / 7 strips bit for bit.  UNet and
pipeline: the product against the CPU oracle at world 3, 5 and 7 and at world 6 with the CFG split (two patch groups of 3),
with the bars of test_unet_gpu.py per step and test_pipeline_gpu.py's for a trajectory.  Ranks share cuda:0 when the box has
fewer GPUs."""
import functools

import pytest
import torch

from helpers import LoopbackArena, _gn_ref, _moments, check_parity, psnr
from mp_product import run_product_trajectory, run_product_unet
from oracle import harness
from oracle.naive_patch import NaiveCase
from oracle.workloads import RaggedCase
from test_ragged_patch_gpu import (_affine, _check, _gn_setup, _i32, _L, _plan, _ragged_attn, _ref, _stream, _weighted_ref,
                                   arenas, sxm_schedule)  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _positions(n):
    return [0, n // 2, n - 1]


# ================================================================================================================ attention
ATTN = [
    # b, lq, lens, own, heads, d: K/V segments of n uneven strips; the tile totals are odd where the K/V range is split in parts
    pytest.param(1, 512, [1408, 1408, 1152], 0, 10, 64, id="n3-own-first-31-tiles"),
    pytest.param(1, 256, [1408, 1300, 1152], 1, 10, 64, id="n3-own-middle-31-tiles"),
    pytest.param(1, 512, [704, 640, 640], 2, 20, 64, id="n3-own-last"),
    pytest.param(1, 256, [700, 640, 640, 520, 512], 0, 10, 64, id="n5-own-first-25-tiles"),
    pytest.param(1, 512, [300, 77, 1000, 640, 257], 2, 8, 40, id="n5-own-middle-d40"),
    pytest.param(1, 640, [640, 640, 640, 512, 512], 4, 4, 160, id="n5-own-last-d160-23-tiles"),
    pytest.param(1, 512, [768, 768, 640, 640, 640, 640], 5, 10, 64, id="n6-own-last"),
    pytest.param(1, 384, [384, 384, 384, 256, 256, 256, 256], 0, 10, 64, id="n7-own-first-17-tiles"),
    pytest.param(1, 2048, [2048, 2048, 2048, 1792, 1792, 1792, 1792], 3, 10, 64, id="n7-own-middle-dynamic"),
    pytest.param(1, 256, [500, 77, 640, 130, 1000, 257, 300], 6, 8, 80, id="n7-own-last-d80"),
]


@pytest.mark.parametrize("b,lq,lens,own,heads,d", ATTN)
def test_attention_any_segment_count(arenas, b, lq, lens, own, heads, d):
    """Attention over 3 / 5 / 6 / 7 unequal segments with the own segment first, in the middle and last, with and without the
    workspace (split K/V parts or the dynamic schedule, and the static whole-unit lists)."""
    torch.manual_seed(53 + sum(lens) + own)
    Cq = heads * d
    segs = [torch.randn(b, x, 2 * Cq, device="cuda", dtype=torch.float16) for x in lens]
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    ref = _ref(q, segs, heads)
    for ws in (True, False):
        out = _ragged_attn(arenas, q, segs, own, heads, d, ws=ws)
        err = (out.float() - ref).abs().max().item()
        assert err < 2e-3, f"workspace={ws}: max abs err {err}"


def test_attention_any_segment_count_schedules(sxm_schedule):
    """The cases above cut odd tile totals into parts (K/V parts that start and end inside a segment) and reach the dynamic
    schedule."""
    tiles = lambda lens: sum(-(-x // 128) for x in lens)
    assert tiles([1408, 1408, 1152]) == 31 and _plan(1, 512, [1408, 1408, 1152], 10, 64) == (40, 3)
    assert tiles([1408, 1300, 1152]) == 31 and _plan(1, 256, [1408, 1300, 1152], 10, 64) == (20, 3)
    assert tiles([700, 640, 640, 520, 512]) == 25 and _plan(1, 256, [700, 640, 640, 520, 512], 10, 64) == (20, 3)
    assert tiles([640, 640, 640, 512, 512]) == 23 and _plan(1, 640, [640, 640, 640, 512, 512], 4, 160) == (20, 2)
    assert tiles([384] * 3 + [256] * 4) == 17 and _plan(1, 384, [384] * 3 + [256] * 4, 10, 64) == (30, 2)
    assert _plan(1, 2048, [2048] * 3 + [1792] * 4, 10, 64) == (160, None)


# ================================================================================================================ GroupNorm
ROWS = {3: [11, 11, 10], 5: [7, 7, 6, 6, 6], 7: [5, 5, 5, 5, 4, 4, 4]}


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("n,rank", [(n, r) for n in (3, 5, 7) for r in _positions(n)])
def test_groupnorm_weighted_any_n(arenas, n, rank, mode):
    """Modes 1 / 2 / 3 with n sources weighted by their rows (SDXL 1024^2 row plans at level 0 / 4 rows per unit)."""
    rows = ROWS[n]
    torch.manual_seed(170 + 8 * n + 4 * mode + rank)
    b, c, w, G = 2, 64, 10, 8
    h = rows[rank]
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    gw, gb = _affine(c)
    arena, now, old, pub, rd = _gn_setup(arenas, mode, rank, n, b, G)
    mean, msq = _weighted_ref(mode, _moments(x, G), now, old, rank, rows)
    y = torch.empty_like(x, memory_format=torch.channels_last)
    scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
    _check(_L().df_groupnorm_fwd_weighted(arena.comm, x.data_ptr(), None, 0, y.data_ptr(), gw.data_ptr(), gb.data_ptr(), b, h, w,
                                          c, G, 1e-5, mode, 1, int(mode == 2), 0, 0, arena.tensor_off[0], arena.slot_bytes[0],
                                          (1 << n) - 1, _i32(rows), scratch.data_ptr(), _stream()), "df_groupnorm_fwd_weighted")
    torch.cuda.synchronize()
    err = (y.float() - _gn_ref(x, G, gw, gb, 1e-5, mean, msq, bessel=True)).abs().max().item()
    assert err < 6e-3, f"max abs err {err}"


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("n,rank", [(n, r) for n in (3, 5, 7) for r in _positions(n)])
def test_groupnorm_halo_weighted_any_n(arenas, n, rank, mode):
    """The fused halo variant: normalised interior, margins from the neighbours (zeros at the image border) and the shipped
    boundary rows, for the first, a middle and the last rank (whose strip is the short one)."""
    rows = ROWS[n]
    torch.manual_seed(190 + 8 * n + 4 * mode + rank)
    b, c, w, G = 2, 64, 10, 8
    h = rows[rank]
    up, down = (rank - 1 if rank > 0 else -1), (rank + 1 if rank < n - 1 else -1)
    hb = 2 * b * w * c * 2
    arena, now, old, pub, rd = _gn_setup(arenas, mode, rank, n, b, G, halo_bytes=hb)
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    gw, gb = _affine(c)
    mean, msq = _weighted_ref(mode, _moments(x, G), now, old, rank, rows)
    top_src, bot_src = torch.randn(b, w, c, device="cuda").half(), torch.randn(b, w, c, device="cuda").half()
    for nbr, part, src in ((up, 1, top_src), (down, 0, bot_src)):
        if nbr >= 0:
            arena.slot(rd, 1, nbr, hb).view(2, b, w, c)[part].copy_(src)
            arena.flags[1, nbr] = rd
    yp = torch.full((b, c, h + 2, w), float("nan"), dtype=torch.float16, device="cuda").contiguous(memory_format=torch.channels_last)
    scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
    _check(_L().df_groupnorm_halo_fwd_weighted(arena.comm, x.data_ptr(), None, 0, yp.data_ptr(), gw.data_ptr(), gb.data_ptr(), b, h,
                                               w, c, G, 1e-5, mode, 1, int(mode == 2), 1, 0, arena.tensor_off[0],
                                               arena.slot_bytes[0], (1 << n) - 1, _i32(rows), scratch.data_ptr(), 1,
                                               arena.tensor_off[1], arena.slot_bytes[1], up, down, 1, 1, _stream()),
           "df_groupnorm_halo_fwd_weighted")
    torch.cuda.synchronize()
    ref = _gn_ref(x, G, gw, gb, 1e-5, mean, msq, bessel=True, silu=True)
    ypn = yp.permute(0, 2, 3, 1)
    err = (ypn[:, 1:-1].float() - ref.permute(0, 2, 3, 1)).abs().max().item()
    assert err < 6e-3, f"max abs err {err}"
    assert torch.equal(ypn[:, 0], top_src if up >= 0 else torch.zeros_like(top_src)), "top margin"
    assert torch.equal(ypn[:, -1], bot_src if down >= 0 else torch.zeros_like(bot_src)), "bottom margin"
    shipped = arena.slot(pub, 1, rank, hb).view(2, b, w, c)
    if up >= 0:
        assert torch.equal(shipped[0], ypn[:, 1])
    if down >= 0:
        assert torch.equal(shipped[1], ypn[:, h])


# ================================================================================================================ halo, publication
POISON = 0x5A


class DistinctArenas:
    """A communicator of n members whose arenas are n separate allocations in this process (same layout), seen from member
    `rank`: a store or flag meant for member p lands in arena p only, so a wrong neighbour or mask bit is visible."""

    def __init__(self, n, slot_bytes, rank):
        from distrifuser_b200 import _lib
        self.members = [LoopbackArena(n, slot_bytes, rank=p) for p in range(n)]
        self.n, self.rank = n, rank
        me = self.members[rank]
        c = _lib.DfComm()
        for p, a in enumerate(self.members):
            c.base[p], c.flags[p] = a.ptr, a.ptr
            a.arena[a.tensor_off[0]:].fill_(POISON)
        c.clock, c.tickets = me.clock.data_ptr(), me.tickets.data_ptr()
        c.bank_stride, c.world, c.rank = me.bank_stride, n, rank
        self.comm, self.me = c, me
        self.before = [a.arena.clone() for a in self.members]

    def expect(self, p, writes):
        """Member p's arena as constructed, with `writes` ((byte offset, uint8 tensor), ...) applied."""
        want = self.before[p].clone()
        for off, data in writes:
            want[off:off + data.numel()] = data
        return want

    def close(self):
        for a in self.members:
            a.close()


def _slot_off(a, epoch, idx, src):
    return (epoch % 3) * a.bank_stride + a.tensor_off[idx] + src * a.slot_bytes[idx]


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8)


def _flag_write(a, idx, src, epoch):
    """(offset, bytes) of flag (idx, src) in a member's flag array holding `epoch`."""
    return 4 * (idx * a.n + src), _bytes(torch.tensor([epoch], dtype=torch.int32, device="cuda"))


@pytest.mark.parametrize("n,rank", [(n, r) for n in (3, 5, 7) for r in _positions(n)])
def test_halo_push_and_assemble_any_n(n, rank):
    """df_halo_push stores this rank's first row into the up neighbour's slot and its last row into the down neighbour's (and
    nothing anywhere else), stamps exactly their flags; df_halo_assemble builds [top halo | x | bottom halo] from them."""
    from distrifuser_b200 import _lib
    L = _lib.lib()
    b, h, w, c, E = 2, 5, 6, 64, 7
    hb = 2 * b * w * c * 2
    up, down = (rank - 1 if rank > 0 else -1), (rank + 1 if rank < n - 1 else -1)
    torch.manual_seed(210 + 8 * n + rank)
    x = torch.randn(b, h, w, c, device="cuda").half()
    ar = DistinctArenas(n, [hb], rank)
    try:
        ar.me.set_clock(pub=E, rd=E - 1)
        _lib.check(L.df_halo_push(ar.comm, x.data_ptr(), b, h, w, c, 0, ar.me.tensor_off[0], ar.me.slot_bytes[0], up, down,
                                  _stream()), "df_halo_push")
        torch.cuda.synchronize()
        for p, a in enumerate(ar.members):
            o = _slot_off(a, E, 0, rank)
            writes = []
            if p == up:                                   # part 0 of this rank's slot: its first row
                writes += [(o, _bytes(x[:, 0])), _flag_write(a, 0, rank, E)]
            if p == down:                                 # part 1: its last row
                writes += [(o + hb // 2, _bytes(x[:, h - 1])), _flag_write(a, 0, rank, E)]
            assert torch.equal(a.arena, ar.expect(p, writes)), f"member {p} (up {up}, down {down})"
        # assemble from the read bank of this rank's own arena
        top_src, bot_src = torch.randn(b, w, c, device="cuda").half(), torch.randn(b, w, c, device="cuda").half()
        for nbr, part, src in ((up, 1, top_src), (down, 0, bot_src)):
            if nbr >= 0:
                ar.me.slot(E - 1, 0, nbr, hb).view(2, b, w, c)[part].copy_(src)
                ar.me.flags[0, nbr] = E - 1
        xp = torch.full((b, h + 2, w, c), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(L.df_halo_assemble(ar.comm, x.data_ptr(), xp.data_ptr(), b, h, w, c, 0, ar.me.tensor_off[0],
                                      ar.me.slot_bytes[0], up, down, 1, _stream()), "df_halo_assemble")
        torch.cuda.synchronize()
        assert torch.equal(xp[:, 1:-1], x)
        assert torch.equal(xp[:, 0], top_src if up >= 0 else torch.zeros_like(top_src))
        assert torch.equal(xp[:, -1], bot_src if down >= 0 else torch.zeros_like(bot_src))
    finally:
        ar.close()


def _masks(n, rank):
    """All peers, every other peer, the last peer."""
    peers = [p for p in range(n) if p != rank]
    return [sum(1 << p for p in peers), sum(1 << p for p in peers[::2]), 1 << peers[-1]]


@pytest.mark.parametrize("strided", [False, True], ids=["contiguous", "strided"])
@pytest.mark.parametrize("n,rank", [(n, r) for n in (3, 5, 7) for r in _positions(n)])
def test_slot_publish_masks_any_n(n, rank, strided):
    """df_slot_publish reaches exactly the members of its mask (all peers, every other peer, one peer): their slot of this
    rank in the publish bank holds the payload and their flag of this rank the epoch; every other byte of every arena is as
    before.  df_slot_wait then returns on the flags of the mask."""
    from distrifuser_b200 import _lib
    L = _lib.lib()
    E, rows, cols = 13, 96, 320
    torch.manual_seed(230 + 8 * n + rank)
    full = torch.randn(rows, 3 * cols, device="cuda").half()
    src = full[:, cols:] if strided else full[:, cols:].contiguous()      # the k|v columns of a fused q|k|v row, or packed
    nbytes = rows * 2 * cols * 2
    for mask in _masks(n, rank):
        ar = DistinctArenas(n, [nbytes], rank)
        try:
            ar.me.set_clock(pub=E, rd=E)
            pitch = src.stride(0) * 2
            _lib.check(L.df_slot_publish(ar.comm, src.data_ptr(), rows, 2 * cols * 2, pitch, ar.me.tensor_off[0],
                                         ar.me.slot_bytes[0], 0, mask, 0, _stream()), "df_slot_publish")
            torch.cuda.synchronize()
            for p, a in enumerate(ar.members):
                writes = [(_slot_off(a, E, 0, rank), _bytes(src)), _flag_write(a, 0, rank, E)] if mask >> p & 1 else []
                assert torch.equal(a.arena, ar.expect(p, writes)), f"mask {mask:#x}: member {p}"
            for s in range(n):
                if mask >> s & 1:
                    ar.me.flags[0, s] = E
            _lib.check(L.df_slot_wait(ar.comm, 0, mask, _stream()), "df_slot_wait")
            torch.cuda.synchronize()
        finally:
            ar.close()


# ================================================================================================================ output gather
def _row_rects(B, H, heights, W):
    """Full-width row strips of the given heights in every batch item (world = B * len(heights), batch-major)."""
    bounds = [sum(heights[:i]) for i in range(len(heights) + 1)]
    assert bounds[-1] == H
    return [(bb, bounds[i], 0, 1, heights[i], W) for bb in range(B) for i in range(len(heights))]


GATHER = {
    # B, C, H, W, rects (batch0, row0, col0, bs, hs, ws) of every world rank, this rank
    "3-rows-uneven": (1, 4, 44, 16, _row_rects(1, 44, [16, 16, 12], 16), 2),
    "5-rows-uneven": (1, 4, 44, 16, _row_rects(1, 44, [12, 8, 8, 8, 8], 16), 0),
    "7-rows-uneven": (1, 4, 36, 12, _row_rects(1, 36, [8, 8, 4, 4, 4, 4, 4], 12), 3),
    "3-cols": (1, 4, 16, 24, [(0, 0, 8 * i, 1, 16, 8) for i in range(3)], 1),
    "5-cols-half": (1, 3, 8, 20, [(0, 0, 4 * i, 1, 8, 4) for i in range(5)], 4),
    "7-cols-half": (1, 3, 6, 21, [(0, 0, 3 * i, 1, 6, 3) for i in range(7)], 6),
    "6-cfg-split-3-rows": (2, 4, 40, 16, _row_rects(2, 40, [16, 12, 12], 16), 4),
}


@pytest.mark.parametrize("name", list(GATHER))
def test_output_gather_any_world(name):
    """The other ranks' strips sit in bank clock[2] (written by the test, flags stamped); this rank scatters its own strip and
    collects the whole image bit for bit.  The banks of the other epochs are poisoned."""
    from distrifuser_b200 import _lib
    B, Cc, H, W, rects, me = GATHER[name]
    n, E = len(rects), 11
    b0, r0, c0, bs, hs, ws = rects[me]
    torch.manual_seed(250 + n)
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
        _lib.check(_lib.lib().df_output_gather_2d(arena.comm, strip.data_ptr(), out.data_ptr(), B, Cc, H, W, bs, hs, ws, b0, r0,
                                                  c0, 0, arena.tensor_off[0], _stream()), "df_output_gather_2d")
        torch.cuda.synchronize()
        assert torch.equal(out, img)
        assert int(arena.flags[0, me].item()) == E
    finally:
        arena.close()


# ================================================================================================================ UNet, pipeline
@pytest.fixture(autouse=True)
def _shared_gpu_timeout(monkeypatch):
    # ranks that time-slice one GPU can stall inside a step for long (cuDNN autotuning in the eager pre-run of 6 processes)
    monkeypatch.setenv("DF_SPIN_TIMEOUT_S", "180")


@functools.lru_cache(maxsize=None)
def _oracle(case, units):
    return harness.run_unet(case, row_units=list(units) if units else None)


UNET = [
    pytest.param(RaggedCase("sdxl_w3", world_size=3, steps=3, lat_h=40), (4, 3, 3), id="sdxl-w3-corrected"),
    pytest.param(RaggedCase("sdxl_w3_full_sync", world_size=3, mode="full_sync", steps=3, lat_h=40), (4, 3, 3),
                 id="sdxl-w3-full_sync"),
    pytest.param(RaggedCase("sdxl_w6_split", world_size=6, split_batch=True, steps=3, lat_h=40), (4, 3, 3), id="sdxl-w6-split-n3"),
    pytest.param(RaggedCase("sd15_w3", family="tiny_sd15", world_size=3, mode="stale_gn", steps=3, lat_h=40, lat_w=24), (2, 2, 1),
                 id="sd15-w3"),
]


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda-graph"])
@pytest.mark.parametrize("case,units", UNET)
def test_unet_any_world(case, units, graph):
    """The product UNet at world 3 (both CFG branches on every rank) and world 6 (two patch groups of 3) against the oracle,
    every step; all ranks agree bit for bit."""
    product = run_product_unet(case, use_graph=graph, row_units=list(units))
    check_parity(case.name, product, _oracle(case, units), ranks_identical=True)


@pytest.mark.parametrize("case,units,graph", [
    pytest.param(RaggedCase("sdxl_w5", world_size=5, steps=3, lat_h=44), [3, 2, 2, 2, 2], False, id="w5-eager"),
    pytest.param(RaggedCase("sdxl_w7", world_size=7, steps=3, lat_h=36), [2, 2, 1, 1, 1, 1, 1], True, id="w7-cuda-graph"),
])
def test_unet_world5_world7(case, units, graph):
    """Five and seven patches (uneven strips, both CFG branches on every rank) against the oracle."""
    product = run_product_unet(case, use_graph=graph, row_units=units)
    check_parity(case.name, product, harness.run_unet(case, row_units=units), ranks_identical=True)


def test_pipeline_trajectory_world3():
    """DistriSDXLPipeline.from_synthetic at 320 x 224 on 3 ranks ([4, 3, 3] units) with CUDA graphs: ranks bit-identical, a
    second image with the same seed identical (checked in the worker), > 35 dB against the oracle trajectory."""
    case = RaggedCase("traj_w3", world_size=3, cfg=True, split_batch=False, warmup_steps=2, lat_h=40)
    got = run_product_trajectory(case, num_steps=8)
    for g in got[1:]:
        assert torch.equal(g, got[0]), "ranks disagree on the final latents"
    want = harness.run_trajectory(case, num_steps=8)
    assert got[0].shape == want.shape == (1, 4, 40, 28)
    p = psnr(got[0], want)
    assert p > 35, f"trajectory PSNR {p:.1f} dB"


def test_naive_patch_world3():
    """Naive patch on 3 ranks, alternate rows / columns with CUDA graphs, at a 36 x 36 latent (strips of 12 whole rows or
    columns) against the naive-patch oracle."""
    case = NaiveCase("naive_sdxl_w3_alternate", world_size=3, scheme="alternate", latent=36)
    check_parity(case.name, run_product_unet(case, use_graph=True), harness.run_unet(case), ranks_identical=True)
