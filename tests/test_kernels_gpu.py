"""GPU parity of each sm_90a kernel through the C ABI, against fp32 torch restatements of the reference math
(oracle/pp_modules.py for the mode formulas).  Tolerances are for fp16 storage with fp32 accumulation:
attention 2e-3 abs on O(1) outputs (P is rounded to fp16 before PV, like every flash kernel), GroupNorm 4e-3
(one fp16 rounding of the output), halo / publication bit-exact."""
import ctypes as C

import pytest
import torch

from helpers import LoopbackArena, _attn, _gn_call, _gn_ref, _moments, _sdpa_ref_chunked, sdpa_ref

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("b,lq,lk,heads,d", [
    (1, 128, 128, 1, 64),          # one tile
    (2, 256, 384, 2, 64),          # multi-tile, multi-head, batch
    (1, 200, 77, 2, 64),           # ragged q tile + cross-attention length (one partial K/V tile)
    (2, 300, 1000, 3, 64),         # ragged both ways, > STAGES tiles
    (1, 1024, 4096, 10, 64),       # SDXL level-1 shape at 1024^2, n=4 (lq=L/4)
    (1, 130, 200, 2, 40),          # SD1.x head_dim 40 (zero-filled to 64 by TMA)
    (2, 300, 520, 2, 80),          # SD1.x head_dim 80  -> two 64-column blocks
    (1, 256, 256, 8, 160),         # SD1.x head_dim 160 -> three 64-column blocks (level 2/3 shape at 1024^2, n=4)
    (1, 64, 256, 2, 160),          # SD1.x deepest level: fewer q rows than one tile
    (1, 200, 77, 2, 80),           # SD1.x cross-attention
    (1, 256, 8192, 4, 64),         # tiny grid, long K/V: 8 K/V parts per unit, merged in-kernel by the last arriver
    (1, 130, 4100, 3, 64),         # split-KV with ragged q and k/v tiles
    (1, 100, 3000, 2, 40),         # split-KV, zero-padded head dim
    (2, 4096, 77, 10, 64),         # persistent CTAs: 640 one-tile work units on 132 resident CTAs (cross-attention at 1024^2 level 1)
    (2, 2048, 300, 20, 64),        # persistent CTAs: 640 units x 3 tiles, ragged last tile
    (2, 1100, 520, 8, 80),         # persistent CTAs, two head blocks: 144 units on 132 CTAs and ragged q
    (2, 2304, 260, 8, 160),        # persistent CTAs, three head blocks: 288 units on 132 CTAs
    (2, 1024, 1024, 20, 64),       # SDXL 1024^2 level 2: 320 units on 132 CTAs (56 CTAs take a third unit)
    (2, 4096, 1024, 10, 64),       # 640 units: four whole units per CTA + 112 left-over units
    (1, 256, 2048, 20, 64),        # 40 units x 16 tiles on 132 slots: 2 K/V parts per unit, merged in-kernel by the last arriver
    (1, 200, 3000, 3, 80),         # split units with two head blocks, ragged q and k/v
])
def test_attention_single_segment(b, lq, lk, heads, d):
    torch.manual_seed(0)
    Cq = heads * d
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16)
    out = _attn(q, kv, heads)
    ref = sdpa_ref(q, kv[..., :Cq], kv[..., Cq:], heads)
    err = (out.float() - ref).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"


@pytest.mark.parametrize("b,lq,lk,heads,d,gain", [(2, 2048, 300, 20, 64, 1.0), (2, 1024, 1024, 20, 64, 30.0), (2, 1100, 520, 8, 80, 1.0)])
def test_attention_static_schedule_without_workspace(b, lq, lk, heads, d, gain):
    """No workspace: every CTA walks its static list of whole units (one case with a large logit jump half-way)."""
    torch.manual_seed(3)
    Cq = heads * d
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16) * (4 if gain > 1 else 1)
    kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16)
    kv[:, lk // 2:, :Cq] *= gain
    out = _attn(q, kv, heads, no_ws=True)
    ref = sdpa_ref(q, kv[..., :Cq], kv[..., Cq:], heads)
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out).all() and err < 4e-3, f"max abs err {err}"


def test_attention_workspace_counters_reset_between_launches():
    """The ticket counter / arrival tickets in the workspace are self-resetting: the same zeroed buffer serves many launches."""
    from distrifuser_b200 import _lib
    torch.manual_seed(5)
    L = _lib.lib()
    b, lq, lk, heads, d = 2, 1024, 1024, 20, 64
    Cq = heads * d
    ws = torch.zeros(L.df_attn_workspace_bytes(b, lq, lk, 1, heads, d), dtype=torch.uint8, device="cuda")
    seg_rank = (C.c_int32 * 8)(*range(8))
    for rep in range(3):
        q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
        kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16)
        out = torch.empty_like(q)
        _lib.check(L.df_attn_fwd(_lib.null_comm(), q.data_ptr(), kv.data_ptr(), out.data_ptr(), None, b, lq, lk, heads, d, q.stride(1),
                                 kv.stride(1), out.stride(1), 1, 0, seg_rank, 0, 0, 0.0, ws.data_ptr(), ws.numel(),
                                 torch.cuda.current_stream().cuda_stream), "df_attn_fwd")
        torch.cuda.synchronize()
        assert int(ws[:4].view(torch.int32).item()) == 0, "ticket counter not reset"
        ref = sdpa_ref(q, kv[..., :Cq], kv[..., Cq:], heads)
        assert (out.float() - ref).abs().max().item() < 2e-3


def test_attention_tail_split_is_planned():
    """df_attn_workspace_bytes: 1 KiB (the ticket counter of the dynamic schedule) unless the schedule also cuts units into K/V
    parts (small grids), which adds the partials."""
    from distrifuser_b200 import _lib
    L = _lib.lib()
    HDR = 1024
    assert L.df_attn_workspace_bytes(1, 256, 8192, 1, 4, 64) > HDR         # 8 units on 132 slots, 64 K/V tiles
    assert L.df_attn_workspace_bytes(2, 1024, 1024, 1, 20, 64) == HDR      # 320 units fill the 132 slots: whole units, dynamic tickets
    assert L.df_attn_workspace_bytes(1, 512, 4096, 1, 10, 64) > HDR        # SDXL 1024^2 n=8 level 1: 40 units x 32 tiles -> 3 parts
    assert L.df_attn_workspace_bytes(2, 1024, 77, 1, 20, 64) == HDR        # cross-attention: one K/V tile, nothing to cut
    assert L.df_attn_workspace_bytes(1, 3600, 3600, 4, 20, 64) == HDR      # 580 units on 132 slots -> whole units


@pytest.mark.parametrize("case", ["late_tiles_x6", "late_tiles_x40", "some_rows", "one_polynomial_column", "one_mufu_column",
                                  "ragged_then_large", "split_parts"])
def test_attention_large_logits_rescale(case):
    """Later K/V tiles whose logits exceed the first tile's by far more than the fp16 head-room of P: the online softmax must
    move the exponent reference and rescale O and l.  The cases cover every row moving, only the rows of one warp moving, the
    jump sitting in a single column that takes the polynomial exp2 or the MUFU exp2, a ragged tile before the jump, and split
    K/V parts."""
    torch.manual_seed(1)
    b, lq, lk, heads, d = 1, 128, 512, 1, 64
    if case == "ragged_then_large":
        lq, lk = 200, 777
    if case == "split_parts":
        lq, lk, heads = 256, 4096, 2          # 4 units on 132 slots: K/V parts merged by the last arriver
    q = torch.randn(b, lq, heads * d, device="cuda", dtype=torch.float16) * 4
    kv = torch.randn(b, lk, 2 * heads * d, device="cuda", dtype=torch.float16)
    C = heads * d
    if case == "late_tiles_x6":
        kv[:, 300:, :C] *= 6
    elif case == "late_tiles_x40":
        kv[:, 130:, :C] *= 40
    elif case == "some_rows":
        q[:, 16:, :] *= 0.1                   # rows 0..15 (one warp's rows) see the jump, the others barely move
        kv[:, 256:, :C] *= 12
    elif case == "one_polynomial_column":
        kv[:, 256 + 3, :C] *= 60              # column 3 of tile 2: group i = 0 -> polynomial lane
    elif case == "one_mufu_column":
        kv[:, 256 + 13, :C] *= 60             # column 13 of tile 2: group i = 1 -> MUFU lane
    elif case == "ragged_then_large":
        kv[:, 640:, :C] *= 10
    elif case == "split_parts":
        kv[:, 1500:, :C] *= 8
        kv[:, 3000:, :C] *= 3
    out = _attn(q, kv, heads)
    ref = sdpa_ref(q, kv[..., :C], kv[..., C:], heads)
    assert torch.isfinite(out).all()
    err = (out.float() - ref).abs().max().item()
    assert err < 4e-3, f"max abs err {err}"


@pytest.mark.parametrize("n,own", [(2, 0), (2, 1), (4, 2)])
def test_attention_multi_segment_stale_slots(n, own):
    """K/V of the peers is read in place from the arena slots of the READ epoch (attn.py:136-138 without the cat)."""
    from distrifuser_b200 import _lib
    torch.manual_seed(2)
    b, lseg, heads, d = 2, 200, 2, 64
    Cq = heads * d
    nbytes = b * lseg * 2 * Cq * 2
    arena = LoopbackArena(n, [nbytes], rank=own)
    epoch = 7
    segs = [torch.randn(b, lseg, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(n)]
    for s in range(n):
        if s != own:
            arena.slot(epoch, 0, s, nbytes).copy_(segs[s].flatten())
            arena.slot(epoch + 1, 0, s, nbytes).fill_(float("nan"))     # a different bank must not be touched
            arena.flags[0, s] = epoch
    arena.set_clock(pub=epoch + 1, rd=epoch)
    maps = torch.empty(_lib.NBANKS * n * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().df_attn_make_kvmaps(arena.comm, arena.tensor_off[0], arena.slot_bytes[0], b, lseg, heads, d,
                                              maps.data_ptr(), torch.cuda.current_stream().cuda_stream), "kvmaps")
    q = torch.randn(b, 300, Cq, device="cuda", dtype=torch.float16)
    out = _attn(q, segs[own], heads, comm=arena.comm, maps=maps.data_ptr(), nseg=n, own=own, lseg=lseg, wait=1)
    full = torch.cat(segs, 1)
    ref = sdpa_ref(q, full[..., :Cq], full[..., Cq:], heads)
    err = (out.float() - ref).abs().max().item()
    arena.close()
    assert err < 2e-3, f"max abs err {err}"


@pytest.mark.parametrize("lq,lseg,heads,own", [(3600, 3600, 20, 1),      # SDXL 3840^2, n=4, level 2 (Lkv 14 400)
                                               (14400, 14400, 10, 3)])   # SDXL 3840^2, n=4, level 1 (Lkv 57 600)
def test_attention_3840_shapes_four_ragged_segments(lq, lseg, heads, own):
    """BASELINE configs[3] per-rank shapes (SURVEY 8a A1): 4 segments whose last tile is ragged (3600 = 28*128 + 16,
    14400 = 112*128 + 64), peers read in place from the arena bank of the read epoch, against a chunked fp32 reference."""
    from distrifuser_b200 import _lib
    torch.manual_seed(11)
    n, b, d = 4, 1, 64
    Cq = heads * d
    nbytes = b * lseg * 2 * Cq * 2
    arena = LoopbackArena(n, [nbytes], rank=own)
    epoch = 4
    segs = [torch.randn(b, lseg, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(n)]
    for s in range(n):
        if s != own:
            arena.slot(epoch, 0, s, nbytes).copy_(segs[s].flatten())
            arena.flags[0, s] = epoch
    arena.set_clock(pub=epoch + 1, rd=epoch)
    maps = torch.empty(_lib.NBANKS * n * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().df_attn_make_kvmaps(arena.comm, arena.tensor_off[0], arena.slot_bytes[0], b, lseg, heads, d,
                                              maps.data_ptr(), torch.cuda.current_stream().cuda_stream), "kvmaps")
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    out = _attn(q, segs[own], heads, comm=arena.comm, maps=maps.data_ptr(), nseg=n, own=own, lseg=lseg, wait=1)
    full = torch.cat(segs, 1)
    ref = _sdpa_ref_chunked(q, full[..., :Cq], full[..., Cq:], heads)
    err = (out.float() - ref).abs().max().item()
    arena.close()
    assert err < 2e-3, f"max abs err {err}"


@pytest.mark.parametrize("B,Cc,H,W,G", [(2, 320, 32, 32, 32), (1, 640, 16, 24, 32), (2, 960, 8, 8, 32), (1, 1280, 15, 60, 32),
                                       (2, 64, 8, 16, 32), (1, 2560, 4, 8, 32), (1, 80, 6, 10, 8), (5, 320, 96, 96, 32)])
@pytest.mark.parametrize("silu", [0, 1])
def test_groupnorm_local(B, Cc, H, W, G, silu):
    from distrifuser_b200 import _lib
    torch.manual_seed(3)
    x = (torch.randn(B, Cc, H, W, device="cuda") * 2 + 0.5).half().contiguous(memory_format=torch.channels_last)
    w = (1 + 0.1 * torch.randn(Cc, device="cuda")).half()
    b_ = (0.1 * torch.randn(Cc, device="cuda")).half()
    y = _gn_call(x, G, w, b_, 1e-5, 0, 0, 0, silu, _lib.null_comm(), 0, 0, 0, 1)
    m, m2 = _moments(x, G)
    ref = _gn_ref(x, G, w, b_, 1e-5, m, m2, bessel=False, silu=bool(silu))
    assert y.is_contiguous(memory_format=torch.channels_last)
    err = (y.float() - ref).abs().max().item()
    assert err < 4e-3 * max(1.0, ref.abs().max().item() / 4), f"max abs err {err}"


def test_groupnorm_fused_addend_twice():
    """GroupNorm(x + t[:, :, None, None]) (ResnetBlock2D time-embedding add) + scratch ticket reuse across calls."""
    from distrifuser_b200 import _lib
    torch.manual_seed(6)
    B, Cc, H, W, G = 2, 640, 16, 16, 32
    x = torch.randn(B, Cc, H, W, device="cuda").half().contiguous(memory_format=torch.channels_last)
    t = torch.randn(B, Cc, device="cuda").half()
    w = (1 + 0.1 * torch.randn(Cc, device="cuda")).half()
    b_ = (0.1 * torch.randn(Cc, device="cuda")).half()
    xs = (x.float() + t.float()[:, :, None, None])
    m, m2 = _moments(xs, G)
    ref = _gn_ref(xs, G, w, b_, 1e-5, m, m2, bessel=False, silu=True)
    for _ in range(2):
        y = _gn_call(x, G, w, b_, 1e-5, 0, 0, 0, 1, _lib.null_comm(), 0, 0, 0, 1, addend=t)
        assert (y.float() - ref).abs().max().item() < 6e-3
    # the addend as a column slice of a wider matrix (the batched time-embedding projection of all ResnetBlock2D): row pitch
    wide = torch.randn(B, 3 * Cc, device="cuda").half()
    wide[:, Cc:2 * Cc] = t
    y = _gn_call(x, G, w, b_, 1e-5, 0, 0, 0, 1, _lib.null_comm(), 0, 0, 0, 1, addend=wide[:, Cc:2 * Cc], apitch=3 * Cc)
    assert (y.float() - ref).abs().max().item() < 6e-3


@pytest.mark.parametrize("mode_name", ["sync", "corrected_async_gn", "stale_gn"])
def test_groupnorm_exchange_modes(mode_name):
    """Mode formulas of groupnorm.py:45-56 with n=2 ranks emulated in one arena (this rank = 0)."""
    torch.manual_seed(4)
    B, Cc, H, W, G, n = 2, 320, 8, 16, 32, 2
    nb = B * G * 8
    arena = LoopbackArena(n, [nb], rank=0)
    w = (1 + 0.1 * torch.randn(Cc, device="cuda")).half()
    b_ = (0.1 * torch.randn(Cc, device="cuda")).half()
    x_now = (torch.randn(B, Cc, H, W, device="cuda") + 0.3).half().contiguous(memory_format=torch.channels_last)
    x_peer = (torch.randn(B, Cc, H, W, device="cuda") * 1.5).half()
    x_old = (torch.randn(B, Cc, H, W, device="cuda") * 0.7 - 0.2).half()      # this rank's previous-step activation
    pack = lambda m, m2: torch.stack([m.flatten(), m2.flatten()], -1).contiguous()
    mine = _moments(x_now, G); peer = _moments(x_peer, G); old = _moments(x_old, G)
    epoch = 5
    if mode_name == "sync":
        arena.slot(epoch, 0, 1, nb, torch.float32).copy_(pack(*peer).flatten())
        arena.flags[0, 1] = epoch
        arena.set_clock(pub=epoch, rd=epoch)
        mode, negfb = 1, 0
        mean, msq = (mine[0] + peer[0]) / 2, (mine[1] + peer[1]) / 2
    else:
        arena.slot(epoch, 0, 1, nb, torch.float32).copy_(pack(*peer).flatten())
        arena.slot(epoch, 0, 0, nb, torch.float32).copy_(pack(*old).flatten())
        arena.flags[0, 0] = epoch; arena.flags[0, 1] = epoch
        arena.set_clock(pub=epoch + 1, rd=epoch)
        if mode_name == "corrected_async_gn":
            mode, negfb = 2, 1
            mean = (old[0] + peer[0]) / 2 + (mine[0] - old[0]); msq = (old[1] + peer[1]) / 2 + (mine[1] - old[1])
            var = msq - mean * mean
            msq = torch.where(var < 0, mine[1] - mine[0] ** 2 + mean * mean, msq)   # groupnorm.py:60-63 as an E[x^2] patch
        else:
            mode, negfb = 3, 0
            mean, msq = (mine[0] + peer[0]) / 2, (mine[1] + peer[1]) / 2
    y = _gn_call(x_now, G, w, b_, 1e-5, mode, 1, negfb, 0, arena.comm, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b11)
    ref = _gn_ref(x_now, G, w, b_, 1e-5, mean, msq, bessel=True)
    err = (y.float() - ref).abs().max().item()
    # the kernel must also have published this step's statistics (slot src=0 of the pub bank) and stamped its flag
    pub = epoch if mode_name == "sync" else epoch + 1
    got = arena.slot(pub, 0, 0, nb, torch.float32).view(B * G, 2)
    pub_err = (got - pack(*mine)).abs().max().item()
    flag = int(arena.flags[0, 0].item())
    arena.close()
    assert err < 6e-3, f"max abs err {err}"
    assert pub_err < 1e-4 and flag == pub


@pytest.mark.parametrize("up,down", [(-1, 1), (0, 2), (2, -1)])
def test_halo_push_and_assemble(up, down):
    from distrifuser_b200 import _lib
    L = _lib.lib()
    torch.manual_seed(5)
    b, c, h, w, n = 2, 64, 6, 10, 4
    rank = 1 if up == 0 else (0 if up < 0 else 3)
    row_bytes = w * c * 2
    arena = LoopbackArena(n, [2 * b * row_bytes], rank=rank)
    x = torch.randn(b, c, h, w, device="cuda").half().contiguous(memory_format=torch.channels_last)
    epoch = 9
    arena.set_clock(pub=epoch, rd=epoch)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.df_halo_push(arena.comm, x.data_ptr(), b, h, w, c, 0, arena.tensor_off[0], arena.slot_bytes[0], up, down, st), "push")
    torch.cuda.synchronize()
    # loopback: what this rank pushed sits in slot src=rank; part 0 = first rows, part 1 = last rows (conv2d.py:90)
    mine = arena.slot(epoch, 0, rank, 2 * b * row_bytes).view(2, b, w, c)
    xn = x.permute(0, 2, 3, 1)                       # [b,h,w,c] view of the NHWC memory
    if up >= 0:
        assert torch.equal(mine[0], xn[:, 0])
    if down >= 0:
        assert torch.equal(mine[1], xn[:, -1])
    # neighbours' rows for the assemble step
    top_src = torch.randn(b, w, c, device="cuda").half()
    bot_src = torch.randn(b, w, c, device="cuda").half()
    if up >= 0:
        arena.slot(epoch, 0, up, 2 * b * row_bytes).view(2, b, w, c)[1].copy_(top_src)
        arena.flags[0, up] = epoch
    if down >= 0:
        arena.slot(epoch, 0, down, 2 * b * row_bytes).view(2, b, w, c)[0].copy_(bot_src)
        arena.flags[0, down] = epoch
    xp = torch.empty((b, c, h + 2, w), dtype=torch.float16, device="cuda", memory_format=torch.channels_last)
    _lib.check(L.df_halo_assemble(arena.comm, x.data_ptr(), xp.data_ptr(), b, h, w, c, 0, arena.tensor_off[0], arena.slot_bytes[0],
                                  up, down, 1, st), "assemble")
    torch.cuda.synchronize()
    xpn = xp.permute(0, 2, 3, 1)
    ok = torch.equal(xpn[:, 1:-1], xn)
    ok &= torch.equal(xpn[:, 0], top_src if up >= 0 else torch.zeros_like(top_src))
    ok &= torch.equal(xpn[:, -1], bot_src if down >= 0 else torch.zeros_like(bot_src))
    arena.close()
    assert ok


@pytest.mark.parametrize("up,down", [(-1, 1), (0, 2), (2, -1)])
@pytest.mark.parametrize("addend", [False, True])
def test_groupnorm_fused_halo(up, down, addend):
    """df_groupnorm_halo_fwd: GroupNorm + SiLU into the interior of the padded conv input, boundary rows shipped to the
    neighbours' slots, margins filled from the neighbours' slots (zeros at the border) -- one kernel instead of
    groupnorm + halo_push + halo_assemble (conv2d.py:72-93)."""
    from distrifuser_b200 import _lib
    L = _lib.lib()
    torch.manual_seed(9)
    b, c, h, w, n, G = 2, 64, 6, 10, 4, 8
    rank = 1 if up == 0 else (0 if up < 0 else 3)
    row_bytes = w * c * 2
    arena = LoopbackArena(n, [b * G * 8, 2 * b * row_bytes], rank=rank)
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    t = torch.randn(b, c, device="cuda").half() if addend else None
    gw = (1 + 0.1 * torch.randn(c, device="cuda")).half()
    gb = (0.1 * torch.randn(c, device="cuda")).half()
    epoch = 9
    arena.set_clock(pub=epoch, rd=epoch)
    top_src = torch.randn(b, w, c, device="cuda").half()
    bot_src = torch.randn(b, w, c, device="cuda").half()
    if up >= 0:
        arena.slot(epoch, 1, up, 2 * b * row_bytes).view(2, b, w, c)[1].copy_(top_src)
        arena.flags[1, up] = epoch
    if down >= 0:
        arena.slot(epoch, 1, down, 2 * b * row_bytes).view(2, b, w, c)[0].copy_(bot_src)
        arena.flags[1, down] = epoch
    yp = torch.full((b, c, h + 2, w), float("nan"), dtype=torch.float16, device="cuda").contiguous(memory_format=torch.channels_last)
    scratch = torch.zeros(L.df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(2):      # twice: the normalise-pass ticket resets itself
        _lib.check(L.df_groupnorm_halo_fwd(arena.comm, x.data_ptr(), t.data_ptr() if addend else None, 0, yp.data_ptr(), gw.data_ptr(),
                                           gb.data_ptr(), b, h, w, c, G, 1e-5, 0, 0, 0, 1, 0, 0, 0, 1, scratch.data_ptr(), 1,
                                           arena.tensor_off[1], arena.slot_bytes[1], up, down, 1, 1, st), "df_groupnorm_halo_fwd")
    torch.cuda.synchronize()
    xs = x.float() + (t.float()[:, :, None, None] if addend else 0.0)
    m, m2 = _moments(xs, G)
    ref = _gn_ref(xs, G, gw, gb, 1e-5, m, m2, bessel=False, silu=True)
    ypn = yp.permute(0, 2, 3, 1)                     # [b, h+2, w, c] view of the NHWC memory
    err = (ypn[:, 1:-1].float() - ref.permute(0, 2, 3, 1)).abs().max().item()
    ok = torch.equal(ypn[:, 0], top_src if up >= 0 else torch.zeros_like(top_src))
    ok &= torch.equal(ypn[:, -1], bot_src if down >= 0 else torch.zeros_like(bot_src))
    mine = arena.slot(epoch, 1, rank, 2 * b * row_bytes).view(2, b, w, c)      # loopback: what this rank shipped
    if up >= 0:
        ok &= torch.equal(mine[0], ypn[:, 1])
    if down >= 0:
        ok &= torch.equal(mine[1], ypn[:, h])
    flag = int(arena.flags[1, rank].item())
    arena.close()
    assert err < 6e-3, f"max abs err {err}"
    assert ok and flag == epoch


def test_publish_and_wait_roundtrip():
    from distrifuser_b200 import _lib
    L = _lib.lib()
    n, nbytes = 4, 3 * 1000 * 256 * 2
    arena = LoopbackArena(n, [nbytes, nbytes], rank=2)
    src = torch.randn(3, 1000, 256, device="cuda").half()
    arena.set_clock(pub=4, rd=4)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.df_slot_publish(arena.comm, src.data_ptr(), 1, nbytes, nbytes, arena.tensor_off[1], arena.slot_bytes[1], 1,
                                 0b1011, 16, st), "publish")
    _lib.check(L.df_slot_wait(arena.comm, 1, 0b0100, st), "wait")      # own flag: set by the publish above
    torch.cuda.synchronize()
    got = arena.slot(4, 1, 2, nbytes).view(3, 1000, 256)
    flag = int(arena.flags[1, 2].item())
    ok = torch.equal(got, src)
    arena.close()
    assert ok and flag == 4


def test_geglu_fused():
    from distrifuser_b200.ops import geglu
    torch.manual_seed(7)
    y = torch.randn(2, 300, 2 * 640, device="cuda").half() * 2
    out = geglu(y)
    h, g = y.float().chunk(2, -1)
    ref = h * torch.nn.functional.gelu(g)
    assert ((out.float() - ref).abs() <= 2e-3 + 2e-3 * ref.abs()).all()      # one fp16 rounding of the product


@pytest.mark.parametrize("C", [320, 640, 1280, 64, 2048])
@pytest.mark.parametrize("with_res", [True, False])
def test_add_layernorm_fused(C, with_res):
    from distrifuser_b200.ops import add_layernorm
    torch.manual_seed(8)
    x = torch.randn(3, 77, C, device="cuda").half()
    r = torch.randn(3, 77, C, device="cuda").half() if with_res else None
    ln = torch.nn.LayerNorm(C).cuda().half()
    with torch.no_grad():
        ln.weight.copy_(1 + 0.1 * torch.randn(C)); ln.bias.copy_(0.1 * torch.randn(C))
    s, y = add_layernorm(x, r, ln)
    s_ref = (x + r) if with_res else x
    assert torch.equal(s, s_ref)
    y_ref = torch.nn.functional.layer_norm(s_ref.float(), (C,), ln.weight.float(), ln.bias.float(), ln.eps)
    assert (y.float() - y_ref).abs().max().item() < 6e-3


def test_publish_strided_rows():
    """k|v columns of a fused q|k|v projection: rows with a pitch larger than the row (df_slot_publish rows > 1)."""
    from distrifuser_b200 import _lib
    L = _lib.lib()
    n, rows, C3 = 2, 3 * 700, 3 * 256
    qkv = torch.randn(rows, C3, device="cuda").half()
    kv = qkv[:, C3 // 3:]
    nbytes = rows * kv.shape[1] * 2
    arena = LoopbackArena(n, [nbytes], rank=0)
    arena.set_clock(pub=2, rd=2)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.df_slot_publish(arena.comm, kv.data_ptr(), rows, kv.shape[1] * 2, C3 * 2, arena.tensor_off[0], arena.slot_bytes[0], 0,
                                 0b10, 16, st), "publish")
    torch.cuda.synchronize()
    got = arena.slot(2, 0, 0, nbytes).view(rows, kv.shape[1])
    ok = torch.equal(got, kv)
    arena.close()
    assert ok


@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("shape", [(2, 320, 16, 24), (1, 1280, 5, 7), (3, 8, 33, 9)])
def test_bias_residual_add(shape, with_res):
    """out = a + bias[c] (+ residual) on NHWC fp16, in place on a: one fp16 rounding of the fp32 sum."""
    from distrifuser_b200 import _lib
    torch.manual_seed(7)
    n, c, h, w = shape
    a = torch.randn(n, c, h, w, device="cuda", dtype=torch.float16).contiguous(memory_format=torch.channels_last)
    r = torch.randn_like(a) if with_res else None
    bias = torch.randn(c, device="cuda", dtype=torch.float16)
    ref = a.float() + bias.float()[None, :, None, None] + (r.float() if with_res else 0)
    _lib.check(_lib.lib().df_bias_residual_add(a.data_ptr(), r.data_ptr() if with_res else None, bias.data_ptr(), a.data_ptr(),
                                               n * h * w, c, torch.cuda.current_stream().cuda_stream), "df_bias_residual_add")
    torch.cuda.synchronize()
    assert torch.equal(a, ref.half())


def test_conv2d_bias_residual_matches_torch():
    """ops.conv2d_bias_residual (cuDNN without bias + one bias / residual pass) against F.conv2d + add."""
    from distrifuser_b200 import ops
    torch.manual_seed(8)
    conv = torch.nn.Conv2d(64, 128, 3, padding=1).cuda().half().to(memory_format=torch.channels_last)
    x = torch.randn(2, 64, 20, 28, device="cuda", dtype=torch.float16).contiguous(memory_format=torch.channels_last)
    res = torch.randn(2, 128, 20, 28, device="cuda", dtype=torch.float16).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        ref = torch.nn.functional.conv2d(x.float(), conv.weight.float(), conv.bias.float(), padding=1) + res.float()
        out = ops.conv2d_bias_residual(x, conv, conv.padding, residual=res)
        out2 = ops.conv2d_bias_residual(x, conv, conv.padding, fold_bias=True) + conv.bias[None, :, None, None] + res
    assert (out.float() - ref).abs().max().item() < 3e-2 and (out2.float() - ref).abs().max().item() < 3e-2
