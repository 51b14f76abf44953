"""GPU parity of patch parallelism on uneven row strips.

Kernels: the attention kernel over K/V segments of unequal length (df_attn_fwd_ragged) and the GroupNorm statistics combine
with per-source weights (df_groupnorm_fwd_weighted / df_groupnorm_halo_fwd_weighted), each against an fp32 torch restatement
at the tolerances of test_kernel_configs_gpu.py; with equal lengths / weights the new entry points must give the bits of the
existing ones.  UNet and pipeline: the product against the CPU oracle on uneven strips (oracle/pp_modules.py), with
test_unet_gpu.py's bars per step and test_pipeline_gpu.py's for a trajectory."""
import ctypes as C

import pytest
import torch

from helpers import LoopbackArena, _gn_ref, _moments, check_parity, psnr, sdpa_ref
from mp_product import run_product_trajectory, run_product_unet
from oracle import harness
from oracle.workloads import RaggedCase

pytestmark = pytest.mark.gpu

BM = BN = 128            # attention: Q rows of a work unit, K/V rows of a tile (csrc/attention.cu)
WS_HEADER = 1024         # attention workspace: ticket counter of the dynamic schedule
MIN_PART_TILES = 8
H100_SMS = 132


def _L():
    from distrifuser_b200 import _lib
    return _lib.lib()


def _check(rc, what):
    from distrifuser_b200 import _lib
    _lib.check(rc, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cdiv(a, b):
    return -(-a // b)


def _i32(values):
    from distrifuser_b200 import _lib
    return _lib.int32_array(values)


@pytest.fixture
def sxm_schedule():
    n = C.c_int(0)
    _check(_L().df_device_sm_count(C.byref(n)), "df_device_sm_count")
    if n.value != H100_SMS:
        pytest.skip(f"schedule expectations are for {H100_SMS} SMs, this device has {n.value}")


@pytest.fixture
def arenas():
    made = []

    def make(n, slot_bytes, rank=0):
        a = LoopbackArena(n, slot_bytes, rank=rank)
        made.append(a)
        return a
    yield make
    for a in made:
        a.close()


# ================================================================================================================ attention
def _plan(b, lq, lens, heads, d):
    """(units, parts) of the schedule: parts = None for the dynamic schedule of a grid that fills the SMs."""
    units = _cdiv(lq, BM) * heads * b
    if units >= H100_SMS:
        return units, None
    tiles = sum(_cdiv(x, BN) for x in lens)
    return units, max(1, min(H100_SMS // units, tiles // MIN_PART_TILES))


def _ws_bytes(units, parts, d):
    if parts is None or parts == 1:
        return WS_HEADER
    hd = _cdiv(d, 64) * 64
    n = units * parts
    return 2 * WS_HEADER + _cdiv(units * 4, 256) * 256 + n * BM * 8 + n * BM * hd * 4


def _ragged_attn(arenas, q, segs, own, heads, d, ws=True, epoch=7):
    """df_attn_fwd_ragged with segs[own] as the own fresh segment and the peers' segments of their own lengths read in place
    from a loopback arena whose slots hold the longest segment (the next bank poisoned with NaN)."""
    from distrifuser_b200 import _lib
    n = len(segs)
    b = q.shape[0]
    lens = [s.shape[1] for s in segs]
    nseg_bytes = [s.numel() * 2 for s in segs]
    arena = arenas(n, [max(nseg_bytes)], rank=own) if n > 1 else None
    maps = None
    comm = _lib.null_comm()
    if n > 1:
        for s in range(n):
            if s != own:
                arena.slot(epoch, 0, s, nseg_bytes[s]).copy_(segs[s].reshape(-1))
                arena.slot(epoch + 1, 0, s, max(nseg_bytes)).fill_(float("nan"))
                arena.flags[0, s] = epoch
        arena.set_clock(pub=epoch + 1, rd=epoch)
        maps = torch.empty(_lib.NBANKS * n * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device="cuda")
        _check(_L().df_attn_make_kvmaps_ragged(arena.comm, arena.tensor_off[0], arena.slot_bytes[0], b, _i32(lens), heads, d,
                                               maps.data_ptr(), _stream()), "df_attn_make_kvmaps_ragged")
        comm = arena.comm
    out = torch.empty(q.shape, dtype=q.dtype, device="cuda")
    ws_bytes = _L().df_attn_workspace_bytes_ragged(b, q.shape[1], _i32(lens), n, heads, d) if ws else 0
    wsb = torch.zeros(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
    _check(_L().df_attn_fwd_ragged(comm, q.data_ptr(), segs[own].data_ptr(), out.data_ptr(),
                                   maps.data_ptr() if maps is not None else None, b, q.shape[1], _i32(lens), heads, d, q.stride(1),
                                   segs[own].stride(1), out.stride(1), n, own, _i32(range(8)), 0, 1, 0.0,
                                   wsb.data_ptr() if ws_bytes else None, ws_bytes, _stream()), "df_attn_fwd_ragged")
    torch.cuda.synchronize()
    return out


def _ref(q, segs, heads):
    full = torch.cat([s.float() for s in segs], 1)
    Cq = q.shape[2]
    return sdpa_ref(q, full[..., :Cq], full[..., Cq:], heads)


RAGGED = [
    # b, lq, lens, own, heads, d: K/V segment lengths of the uneven strips' tokens
    pytest.param(1, 512, [512, 500, 450, 512], 1, 10, 64, id="under-a-tile-d64"),     # lengths differ by < 1 tile
    pytest.param(1, 512, [1000, 77, 640, 300], 2, 10, 64, id="several-tiles-d64"),    # 1-tile segment, middle tails
    pytest.param(1, 512, [300, 77, 1000, 640], 0, 8, 40, id="several-tiles-d40"),
    pytest.param(1, 1024, [700, 1100, 128, 260], 3, 8, 80, id="several-tiles-d80"),
    pytest.param(1, 256, [384, 257, 130], 1, 4, 160, id="tail-tiles-d160"),
    pytest.param(1, 2048, [2048, 1664, 1664, 1664], 0, 10, 64, id="dynamic-schedule"),            # fills the SMs
    pytest.param(1, 512, [512, 384], 1, 20, 64, id="n2-5-4-units-level2"),
]


@pytest.mark.parametrize("b,lq,lens,own,heads,d", RAGGED)
def test_attention_unequal_segments(sxm_schedule, arenas, b, lq, lens, own, heads, d):
    """Attention over the concatenation of unequal segments: tail masks at each segment's own length, split K/V parts over
    the total tile count (and the dynamic schedule where the grid fills the SMs); with and without the workspace."""
    units, parts = _plan(b, lq, lens, heads, d)
    got_ws = _L().df_attn_workspace_bytes_ragged(b, lq, _i32(lens), len(lens), heads, d)
    assert got_ws == _ws_bytes(units, parts, d), f"expected plan units={units} parts={parts}, workspace {got_ws}"
    torch.manual_seed(41 + sum(lens))
    Cq = heads * d
    segs = [torch.randn(b, x, 2 * Cq, device="cuda", dtype=torch.float16) for x in lens]
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    ref = _ref(q, [segs[(own + o) % len(segs)] for o in range(len(segs))], heads)   # order does not matter to softmax
    for ws in (True, False):
        out = _ragged_attn(arenas, q, segs, own, heads, d, ws=ws)
        err = (out.float() - ref).abs().max().item()
        assert err < 2e-3, f"workspace={ws}: max abs err {err}"


def test_attention_schedules_reached(sxm_schedule):
    """The cases above reach both schedules: split K/V parts (units < SMs) and the dynamic ticket schedule."""
    assert _plan(1, 512, [512, 500, 450, 512], 10, 64) == (40, 2)
    assert _plan(1, 512, [1000, 77, 640, 300], 10, 64)[1] == 2
    assert _plan(1, 2048, [2048, 1664, 1664, 1664], 10, 64) == (160, None)


@pytest.mark.parametrize("lq,lseg,nseg,own,heads,d", [
    (4096, 4096, 1, 0, 10, 64), (1024, 1024, 1, 0, 20, 64),               # bench shapes, one segment
    (512, 512, 8, 5, 10, 64), (1024, 1024, 4, 3, 8, 80), (512, 500, 8, 3, 10, 64), (256, 256, 2, 1, 4, 160),
])
def test_attention_ragged_entry_points_equal_lengths_bit_identical(arenas, lq, lseg, nseg, own, heads, d):
    """Equal lengths through df_attn_make_kvmaps_ragged / df_attn_workspace_bytes_ragged / df_attn_fwd_ragged give the bits of
    df_attn_make_kvmaps / df_attn_workspace_bytes / df_attn_fwd."""
    from helpers import _attn
    from distrifuser_b200 import _lib
    b = 1
    torch.manual_seed(lq + nseg)
    Cq = heads * d
    segs = [torch.randn(b, lseg, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(nseg)]
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    assert _L().df_attn_workspace_bytes(b, lq, lseg, nseg, heads, d) == \
        _L().df_attn_workspace_bytes_ragged(b, lq, _i32([lseg] * nseg), nseg, heads, d)
    new = _ragged_attn(arenas, q, segs, own, heads, d)
    if nseg == 1:
        old = _attn(q, segs[0], heads, d=d)
    else:
        nbytes = segs[0].numel() * 2
        arena = arenas(nseg, [nbytes], rank=own)
        for s in range(nseg):
            if s != own:
                arena.slot(7, 0, s, nbytes).copy_(segs[s].reshape(-1))
                arena.flags[0, s] = 7
        arena.set_clock(pub=8, rd=7)
        maps = torch.empty(_lib.NBANKS * nseg * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device="cuda")
        _check(_L().df_attn_make_kvmaps(arena.comm, arena.tensor_off[0], arena.slot_bytes[0], b, lseg, heads, d, maps.data_ptr(),
                                        _stream()), "df_attn_make_kvmaps")
        old = _attn(q, segs[own], heads, comm=arena.comm, maps=maps.data_ptr(), nseg=nseg, own=own, lseg=lseg, wait=1, d=d)
    assert torch.equal(new, old)


# ================================================================================================================ GroupNorm
def _pack(m, m2):
    return torch.stack([m.flatten(), m2.flatten()], -1).contiguous()


def _fake_moments(B, G):
    m = 0.3 * torch.randn(B, G, 1, 1, 1, device="cuda")
    return m, m * m + 0.5 + torch.rand(B, G, 1, 1, 1, device="cuda")


def _affine(Cc):
    return (1 + 0.1 * torch.randn(Cc, device="cuda")).half(), (0.1 * torch.randn(Cc, device="cuda")).half()


def _gn_setup(arenas, mode, rank, n, b, G, halo_bytes=None):
    """Statistics in a loopback arena inside an asynchronous step (pub = e + 1, rd = e): `now` (mode 1) and `old` (modes 2, 3)."""
    e = 9
    pub, rd = e + 1, e
    nb = b * G * 8
    arena = arenas(n, [nb] + ([halo_bytes] if halo_bytes else []), rank=rank)
    now = [_fake_moments(b, G) for _ in range(n)]
    old = [_fake_moments(b, G) for _ in range(n)]
    for s in range(n):
        arena.slot(rd, 0, s, nb, torch.float32).copy_(_pack(*old[s]).flatten())
        if s != rank:
            arena.slot(pub, 0, s, nb, torch.float32).copy_(_pack(*now[s]).flatten())
        arena.flags[0, s] = pub if (mode == 1 and s != rank) else rd
    arena.set_clock(pub=pub, rd=rd)
    return arena, now, old, pub, rd


def _weighted_ref(mode, mine, now, old, rank, rows):
    wts = [r / sum(rows) for r in rows]
    if mode == 1:
        src = [mine if s == rank else now[s] for s in range(len(rows))]
        return sum(w * m[0] for w, m in zip(wts, src)), sum(w * m[1] for w, m in zip(wts, src))
    if mode == 2:
        return (sum(w * o[0] for w, o in zip(wts, old)) + (mine[0] - old[rank][0]),
                sum(w * o[1] for w, o in zip(wts, old)) + (mine[1] - old[rank][1]))
    src = [mine if s == rank else old[s] for s in range(len(rows))]
    return sum(w * m[0] for w, m in zip(wts, src)), sum(w * m[1] for w, m in zip(wts, src))


@pytest.mark.parametrize("rows,rank", [([12, 8, 8, 8], 0), ([12, 8, 8, 8], 2), ([10, 8], 1), ([2, 1, 1, 1], 3)])
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_groupnorm_weighted_modes(arenas, mode, rows, rank):
    """Modes 1 / 2 / 3 with each source weighted by its share of the rows (integers reduced by their gcd in the kernel)."""
    torch.manual_seed(70 + 4 * mode + rank)
    n, b, c, w, G = len(rows), 2, 64, 10, 8
    h = rows[rank]
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    gw, gb = _affine(c)
    arena, now, old, pub, rd = _gn_setup(arenas, mode, rank, n, b, G)
    mine = _moments(x, G)
    mean, msq = _weighted_ref(mode, mine, now, old, rank, rows)
    assert (msq - mean * mean).min().item() > 0.1
    y = torch.empty_like(x, memory_format=torch.channels_last)
    scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
    _check(_L().df_groupnorm_fwd_weighted(arena.comm, x.data_ptr(), None, 0, y.data_ptr(), gw.data_ptr(), gb.data_ptr(), b, h, w,
                                          c, G, 1e-5, mode, 1, int(mode == 2), 0, 0, arena.tensor_off[0], arena.slot_bytes[0],
                                          (1 << n) - 1, _i32(rows), scratch.data_ptr(), _stream()), "df_groupnorm_fwd_weighted")
    torch.cuda.synchronize()
    ref = _gn_ref(x, G, gw, gb, 1e-5, mean, msq, bessel=True)
    err = (y.float() - ref).abs().max().item()
    assert err < 6e-3, f"max abs err {err}"
    # the 1/n combine is measurably different here: the weights are what the kernel used
    m1, q1 = _weighted_ref(mode, mine, now, old, rank, [1] * n)
    wrong = _gn_ref(x, G, gw, gb, 1e-5, m1, q1, bessel=True)
    assert (wrong - ref).abs().max().item() > 3e-2


@pytest.mark.parametrize("rank", [0, 1, 3])
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_groupnorm_halo_weighted(arenas, mode, rank):
    """The fused halo variant with weights [3, 2, 2, 2] (rows 6 / 4 / 4 / 4): normalised interior, shipped rows and margins."""
    rows = [6, 4, 4, 4]
    torch.manual_seed(90 + 4 * mode + rank)
    n, b, c, w, G = 4, 2, 64, 10, 8
    h = rows[rank]
    up, down = (rank - 1 if rank > 0 else -1), (rank + 1 if rank < n - 1 else -1)
    hb = 2 * b * w * c * 2
    arena, now, old, pub, rd = _gn_setup(arenas, mode, rank, n, b, G, halo_bytes=hb)
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    gw, gb = _affine(c)
    mine = _moments(x, G)
    mean, msq = _weighted_ref(mode, mine, now, old, rank, rows)
    top_src, bot_src = torch.randn(b, w, c, device="cuda").half(), torch.randn(b, w, c, device="cuda").half()
    for nbr, part, src in ((up, 1, top_src), (down, 0, bot_src)):
        if nbr >= 0:
            arena.slot(rd, 1, nbr, hb).view(2, b, w, c)[part].copy_(src)
            arena.flags[1, nbr] = rd
    yp = torch.full((b, c, h + 2, w), float("nan"), dtype=torch.float16, device="cuda").contiguous(memory_format=torch.channels_last)
    scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
    _check(_L().df_groupnorm_halo_fwd_weighted(arena.comm, x.data_ptr(), None, 0, yp.data_ptr(), gw.data_ptr(), gb.data_ptr(), b, h,
                                               w, c, G, 1e-5, mode, 1, int(mode == 2), 1, 0, arena.tensor_off[0],
                                               arena.slot_bytes[0], 0b1111, _i32(rows), scratch.data_ptr(), 1, arena.tensor_off[1],
                                               arena.slot_bytes[1], up, down, 1, 1, _stream()), "df_groupnorm_halo_fwd_weighted")
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


@pytest.mark.parametrize("halo", [False, True])
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_groupnorm_weighted_equal_weights_bit_identical(arenas, mode, halo):
    """Equal weights (any common value: reduced by the gcd to 1) give the bits of df_groupnorm_fwd / df_groupnorm_halo_fwd."""
    torch.manual_seed(110 + mode)
    n, rank, b, c, h, w, G = 4, 1, 2, 320, 8, 12, 32
    hb = 2 * b * w * c * 2
    arena, now, old, pub, rd = _gn_setup(arenas, mode, rank, n, b, G, halo_bytes=hb)
    for s in (0, 2):
        arena.flags[1, s] = rd
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    gw, gb = _affine(c)
    outs = []
    for weights in (None, [5, 5, 5, 5]):
        yp = torch.empty((b, c, h + 2 if halo else h, w), dtype=torch.float16, device="cuda").contiguous(memory_format=torch.channels_last)
        scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
        args = (arena.comm, x.data_ptr(), None, 0, yp.data_ptr(), gw.data_ptr(), gb.data_ptr(), b, h, w, c, G, 1e-5, mode, 1,
                int(mode == 2), 1, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b1111)
        tail = (1, arena.tensor_off[1], arena.slot_bytes[1], 0, 2, 0, 1, _stream()) if halo else (_stream(),)
        if weights is None:
            fn = _L().df_groupnorm_halo_fwd if halo else _L().df_groupnorm_fwd
            _check(fn(*args, scratch.data_ptr(), *tail), "df_groupnorm_fwd")
        else:
            fn = _L().df_groupnorm_halo_fwd_weighted if halo else _L().df_groupnorm_fwd_weighted
            _check(fn(*args, _i32(weights), scratch.data_ptr(), *tail), "df_groupnorm_fwd_weighted")
        torch.cuda.synchronize()
        outs.append(yp.clone())
    assert torch.equal(outs[0], outs[1])


# ================================================================================================================ UNet, pipeline
MODES = ("corrected_async_gn", "stale_gn", "sync_gn", "separate_gn", "full_sync", "no_sync")
UNET = [pytest.param(RaggedCase(f"sdxl_n2_{m}", world_size=2, mode=m, steps=3), [5, 4], False, id=f"n2-{m}") for m in MODES] + [
    pytest.param(RaggedCase("sdxl_n4", world_size=4, steps=3), [3, 2, 2, 2], False, id="n4-nosplit"),
    pytest.param(RaggedCase("sd15_n4", family="tiny_sd15", world_size=4, mode="stale_gn", steps=3, lat_h=40, lat_w=24),
                 [2, 1, 1, 1], False, id="sd15-n4-2111"),
    pytest.param(RaggedCase("sdxl_n2_graph", world_size=2, steps=3), [5, 4], True, id="n2-cuda-graph"),
]


@pytest.mark.parametrize("case,units,graph", UNET)
def test_unet_uneven_strips(case, units, graph):
    """The product UNet over uneven strips against the uneven oracle, every step; all ranks agree bit for bit."""
    product = run_product_unet(case, use_graph=graph, row_units=units)
    check_parity(case.name, product, harness.run_unet(case, row_units=units), ranks_identical=True)


@pytest.mark.multigpu(8)
def test_unet_uneven_strips_eight_gpus():
    """cfg2 x patch4 over [3, 2, 2, 2] units on 8 real GPUs."""
    case = RaggedCase("sdxl_w8_split", world_size=8, split_batch=True, steps=3)
    product = run_product_unet(case, row_units=[3, 2, 2, 2])
    check_parity(case.name, product, harness.run_unet(case, row_units=[3, 2, 2, 2]), ranks_identical=True)


def test_pipeline_uneven_height_trajectory():
    """DistriSDXLPipeline.from_synthetic at 288 x 224 on 2 ranks ([5, 4] units) with CUDA graphs: ranks bit-identical, a
    second image with the same seed identical (checked in the worker), > 35 dB against the oracle trajectory."""
    case = RaggedCase("traj", world_size=2, cfg=True, split_batch=False, warmup_steps=2)
    got = run_product_trajectory(case, num_steps=8)
    for g in got[1:]:
        assert torch.equal(g, got[0]), "ranks disagree on the final latents"
    want = harness.run_trajectory(case, num_steps=8)
    assert got[0].shape == want.shape == (1, 4, 36, 28)
    p = psnr(got[0], want)
    assert p > 35, f"trajectory PSNR {p:.1f} dB"
