"""GPU parity of the sm_90a kernels at the launch configurations the product uses: the attention kernel's split K/V schedule
over several peer segments (the 8-GPU plans of SD1.5 / SDXL at 1024^2), the strided q | k | v views of the fused projection,
zero-padded heads with an explicit softmax scale, every head width of the NBLK blocks; GroupNorm exchange modes inside an
asynchronous step, the negative-variance fallback, the fused halo with statistics exchange and edge shapes; the output gather
and the epoch clock; the GEMM's forced tile widths, CTA caps, pitched output / residual and fused publication.  References
are fp32 (fp64 where noted) torch restatements of the same math; tolerances as in test_kernels_gpu.py / test_linear_gpu.py.
Every test first asserts that it reaches the path it is about."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from helpers import LoopbackArena, _attn, _close, _gn_call, _gn_ref, _moments, sdpa_ref

pytestmark = pytest.mark.gpu

BM = BN = 128            # attention: Q rows of a work unit, K/V rows of a tile (csrc/attention.cu)
WS_HEADER = 1024         # attention workspace: ticket counter of the dynamic schedule
MIN_PART_TILES = 8       # attention: a part of a split unit keeps at least this many K/V tiles
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


@pytest.fixture
def sxm_schedule():
    """The schedules pinned below (units per SM slot, parts per unit) are those of a 132-SM H100 SXM."""
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
def _split_ws_bytes(units, parts, d):
    """df_attn_workspace_bytes of a plan that cuts each of `units` work units into `parts` K/V ranges (workspace_need):
    header, 1 KiB, arrival tickets (256-byte rounded), fp32 (m, l) and O partials of 128 rows per part."""
    hd = _cdiv(d, 64) * 64
    n = units * parts
    return 2 * WS_HEADER + _cdiv(units * 4, 256) * 256 + n * BM * 8 + n * BM * hd * 4


def _assert_plan(b, lq, lseg, nseg, heads, d, P):
    """P = None: a grid that fills the SMs (dynamic ticket schedule, header-only workspace); else units cut into P parts."""
    units = _cdiv(lq, BM) * heads * b
    got = _L().df_attn_workspace_bytes(b, lq, lseg, nseg, heads, d)
    if P is None:
        assert units >= H100_SMS and got == WS_HEADER, f"expected the dynamic schedule: {units} units, workspace {got}"
    else:
        assert units < H100_SMS and got == _split_ws_bytes(units, P, d), \
            f"expected {units} units in {P} parts ({_split_ws_bytes(units, P, d)} B), workspace is {got} B"
    return units


def _peer_arena(arenas, segs, own, heads, d, epoch=7):
    """The peers' K/V segments (s != own) in the arena bank of the read epoch with their flags stamped, the next bank
    poisoned with NaN; returns (arena, tensor maps)."""
    from distrifuser_b200 import _lib
    n = len(segs)
    b, lseg, w2 = segs[own].shape
    nbytes = b * lseg * w2 * 2
    arena = arenas(n, [nbytes], rank=own)
    for s in range(n):
        if s != own:
            arena.slot(epoch, 0, s, nbytes).copy_(segs[s].reshape(-1))
            arena.slot(epoch + 1, 0, s, nbytes).fill_(float("nan"))
            arena.flags[0, s] = epoch
    arena.set_clock(pub=epoch + 1, rd=epoch)
    maps = torch.empty(_lib.NBANKS * n * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device="cuda")
    _check(_L().df_attn_make_kvmaps(arena.comm, arena.tensor_off[0], arena.slot_bytes[0], b, lseg, heads, d, maps.data_ptr(),
                                    _stream()), "df_attn_make_kvmaps")
    return arena, maps


def _attn_segs(q, segs, own, heads, arenas, d=None, **kw):
    """df_attn_fwd with this rank's segment segs[own] and the peers' read in place from a loopback arena."""
    d = d or q.shape[2] // heads
    if len(segs) == 1:
        return _attn(q, segs[0], heads, d=d, **kw)
    arena, maps = _peer_arena(arenas, segs, own, heads, d)
    return _attn(q, segs[own], heads, comm=arena.comm, maps=maps.data_ptr(), nseg=len(segs), own=own, lseg=segs[own].shape[1],
                 wait=1, d=d, **kw)


def _ref_segs(q, segs, heads):
    full = torch.cat([s.float() for s in segs], 1)
    Cq = q.shape[2]
    return sdpa_ref(q, full[..., :Cq], full[..., Cq:], heads)


@pytest.mark.parametrize("b,lq,lseg,heads,d,nseg,own,P", [
    pytest.param(1, 1024, 1024, 8, 80, 4, 0, 2, id="sd15-1024-n8-level1-own0"),     # BASELINE configs[4], level 1
    pytest.param(1, 1024, 1024, 8, 80, 4, 3, 2, id="sd15-1024-n8-level1-own3"),
    pytest.param(1, 512, 512, 10, 64, 8, 0, 3, id="sdxl-1024-n8-level1-own0"),      # parts start at tiles 10 and 21
    pytest.param(1, 512, 512, 10, 64, 8, 5, 3, id="sdxl-1024-n8-level1-own5"),
    pytest.param(1, 512, 512, 10, 64, 8, 7, 3, id="sdxl-1024-n8-level1-own7"),
    pytest.param(1, 512, 500, 10, 64, 8, 3, 3, id="ragged-lseg500-own3"),           # parts start mid-segment, last tiles ragged
])
def test_attention_multi_segment_split_kv(sxm_schedule, arenas, b, lq, lseg, heads, d, nseg, own, P):
    """Split K/V ranges over several segments: parts start mid-segment, wrap past the last segment to segment 0 and take the
    first-tile flag wait.  With the workspace (split plan) and without it (static whole units): both against the reference
    and against each other."""
    _assert_plan(b, lq, lseg, nseg, heads, d, P)
    tps = _cdiv(lseg, BN)
    starts = [p * nseg * tps // P for p in range(P)]
    assert P <= nseg * tps // MIN_PART_TILES and starts == ([0, 16] if P == 2 else [0, 10, 21]), f"parts start at tiles {starts}"
    torch.manual_seed(12)
    Cq = heads * d
    segs = [torch.randn(b, lseg, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(nseg)]
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    ref = _ref_segs(q, segs, heads)
    split = _attn_segs(q, segs, own, heads, arenas)
    whole = _attn_segs(q, segs, own, heads, arenas, no_ws=True)
    for name, out in (("split", split), ("whole units", whole)):
        err = (out.float() - ref).abs().max().item()
        assert err < 2e-3, f"{name}: max abs err {err}"
    assert (split.float() - whole.float()).abs().max().item() < 2e-3


def test_attention_split_parts_large_logit_gaps(sxm_schedule, arenas):
    """SDXL n=8 plan (3 parts of 10 / 11 / 11 tiles): one peer segment's K scaled by 30 puts the maximum in part 2, part 1's
    merge weight 2^(m_1 - m_max) is below 2^-20, and the segments of part 0 have logits so far below that its weight
    underflows to 0."""
    b, lq, lseg, heads, d, nseg, own, P = 1, 512, 512, 10, 64, 8, 0, 3
    _assert_plan(b, lq, lseg, nseg, heads, d, P)
    torch.manual_seed(13)
    Cq = heads * d
    q = (0.25 * torch.randn(b, lq, Cq, device="cuda") + 0.5).half()              # mostly positive: sign-stable logits
    segs = [torch.randn(b, lseg, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(nseg)]
    for s in (0, 1, 2):
        segs[s][..., :Cq] = (-24 + 0.1 * torch.randn(b, lseg, Cq, device="cuda")).half()
    segs[6][..., :Cq] *= 30
    # precondition: per-row maxima of every part (log2 units), keys in segment order own, own + 1, ... (own = 0)
    k = torch.cat([s[..., :Cq] for s in segs], 1).float().view(b, -1, heads, d).transpose(1, 2)
    qh = q.float().view(b, lq, heads, d).transpose(1, 2)
    s2 = (qh @ k.transpose(-1, -2)) * (d ** -0.5) * 1.4426950408889634
    T = nseg * _cdiv(lseg, BN)
    bounds = [p * T // P * BN for p in range(P + 1)]
    m = torch.stack([s2[..., bounds[p]:bounds[p + 1]].amax(-1) for p in range(P)])
    gap = m - m.amax(0)
    assert (gap[2] == 0).all(), "the scaled segment must hold every row's maximum"
    assert gap[1].max().item() < -20, f"part 1 weight not small: {gap[1].max().item()}"
    assert gap[0].max().item() < -130, f"part 0 weight does not underflow: {gap[0].max().item()}"
    out = _attn_segs(q, segs, own, heads, arenas)
    ref = _ref_segs(q, segs, heads)
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out).all() and err < 4e-3, f"max abs err {err}"


@pytest.mark.parametrize("b,l,heads,d,nseg,own,P", [
    pytest.param(2, 1024, 20, 64, 1, 0, None, id="d64-dynamic"),
    pytest.param(1, 512, 10, 64, 8, 5, 3, id="d64-n8-split"),
    pytest.param(2, 2304, 8, 160, 1, 0, None, id="d160-dynamic"),
    pytest.param(1, 512, 8, 160, 4, 1, 2, id="d160-n4-split"),
])
def test_attention_fused_qkv_layout(sxm_schedule, arenas, b, l, heads, d, nseg, own, P):
    """Self-attention as the product calls it: q and this rank's k|v are column views of one [b, l, 3C] projection (row pitch
    3C) and the output is a column slice of a wider buffer; the columns outside the slice stay untouched."""
    _assert_plan(b, l, l, nseg, heads, d, P)
    torch.manual_seed(14)
    Cq = heads * d
    qkv = torch.randn(b, l, 3 * Cq, device="cuda", dtype=torch.float16)
    q, kv = qkv[..., :Cq], qkv[..., Cq:]
    assert q.stride(1) == kv.stride(1) == 3 * Cq
    segs = [torch.randn(b, l, 2 * Cq, device="cuda", dtype=torch.float16) for _ in range(nseg)]
    segs[own] = kv
    wide = torch.full((b, l, Cq + 24), 7.0, device="cuda", dtype=torch.float16)
    out = wide[..., 8:8 + Cq]
    _attn_segs(q, segs, own, heads, arenas, out=out)
    ref = _ref_segs(q, segs, heads)
    err = (out.float() - ref).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"
    assert (wide[..., :8] == 7).all() and (wide[..., 8 + Cq:] == 7).all(), "columns outside the output slice were written"


@pytest.mark.parametrize("b,l,nseg,own,P", [pytest.param(2, 2048, 1, 0, None, id="dynamic"),
                                            pytest.param(1, 512, 4, 2, 2, id="n4-split")])
def test_attention_zero_padded_heads_explicit_scale(sxm_schedule, arenas, b, l, nseg, own, P):
    """SD1.5 level 0: heads of 40 stored 64 wide (zero columns 40..63 in q, k and v) with scale = 40^-0.5 passed explicitly,
    q | k | v as views of one projection.  Against the reference on the compact 40-wide heads; the padding columns of the
    output are exactly 0."""
    heads, dr, dp = 8, 40, 64
    _assert_plan(b, l, l, nseg, heads, dp, P)
    torch.manual_seed(15)

    def padded(*parts):              # compact [b, l, heads*40] tensors -> [b, l, len(parts) * heads*64], zero-padded heads
        t = torch.zeros(b, l, len(parts), heads, dp, device="cuda", dtype=torch.float16)
        t[..., :dr] = torch.stack(parts, 2).view(b, l, len(parts), heads, dr)
        return t.view(b, l, len(parts) * heads * dp)

    comp = [[torch.randn(b, l, heads * dr, device="cuda", dtype=torch.float16) for _ in range(2)] for _ in range(nseg)]
    qc = torch.randn(b, l, heads * dr, device="cuda", dtype=torch.float16)
    qkv = padded(qc, *comp[own])
    Cs = heads * dp
    segs = [padded(*c) for c in comp]
    segs[own] = qkv[..., Cs:]
    out = _attn_segs(qkv[..., :Cs], segs, own, heads, arenas, d=dp, scale=dr ** -0.5)
    kc = torch.cat([c[0] for c in comp], 1)
    vc = torch.cat([c[1] for c in comp], 1)
    ref = sdpa_ref(qc, kc, vc, heads).view(b, l, heads, dr)
    o = out.view(b, l, heads, dp)
    err = (o[..., :dr].float() - ref).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"
    assert (o[..., dr:] == 0).all(), "padding columns of the output are not zero"


@pytest.mark.parametrize("d", [8, 16, 56, 64, 72, 120, 128, 136, 184, 192])
def test_attention_head_dim_sweep(d):
    """Every head width class: one / two / three 64-column blocks and both sides of each block boundary, ragged q and k/v."""
    torch.manual_seed(16)
    b, lq, lk, heads = 2, 200, 333, 3
    Cq = heads * d
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
    kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16)
    out = _attn(q, kv, heads)
    err = (out.float() - sdpa_ref(q, kv[..., :Cq], kv[..., Cq:], heads)).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"


def test_attention_head_dim_192_multi_segment(arenas):
    torch.manual_seed(17)
    b, lq, lseg, heads, d, nseg, own = 1, 300, 200, 2, 192, 3, 1
    segs = [torch.randn(b, lseg, 2 * heads * d, device="cuda", dtype=torch.float16) for _ in range(nseg)]
    q = torch.randn(b, lq, heads * d, device="cuda", dtype=torch.float16)
    out = _attn_segs(q, segs, own, heads, arenas)
    err = (out.float() - _ref_segs(q, segs, heads)).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"


def test_attention_one_workspace_across_shapes(sxm_schedule):
    """One zeroed workspace serves launches of different plans back to back (as the per-device shared workspace serves every
    layer): split -> dynamic -> another split -> the first split again.  The ticket word and the arrival tickets are zero
    after every launch."""
    shapes = [(1, 256, 8192, 4, 64, 8), (2, 1024, 1024, 20, 64, None), (1, 512, 4096, 10, 64, 3), (1, 256, 8192, 4, 64, 8)]
    need = [_L().df_attn_workspace_bytes(b, lq, lk, 1, h, d) for b, lq, lk, h, d, _ in shapes]
    ws = torch.zeros(max(need), dtype=torch.uint8, device="cuda")
    torch.manual_seed(18)
    for b, lq, lk, heads, d, P in shapes:
        units = _assert_plan(b, lq, lk, 1, heads, d, P)
        Cq = heads * d
        q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16)
        kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16)
        out = _attn(q, kv, heads, ws=ws)
        err = (out.float() - sdpa_ref(q, kv[..., :Cq], kv[..., Cq:], heads)).abs().max().item()
        assert err < 2e-3, f"shape {(b, lq, lk, heads, d)}: max abs err {err}"
        assert int(ws[:4].view(torch.int32).item()) == 0, "ticket counter not reset"
        assert P is None or units * 4 <= 256, "the arrival tickets checked below must cover every unit"
        assert not ws[WS_HEADER:WS_HEADER + 256].any(), "arrival tickets not reset"


# ================================================================================================================ GroupNorm
def _pack(m, m2):
    return torch.stack([m.flatten(), m2.flatten()], -1).contiguous()


def _fake_moments(B, G, seed_scale=1.0):
    """Finite statistics of a plausible activation: (E[x], E[x^2]) with a positive variance."""
    m = 0.3 * seed_scale * torch.randn(B, G, 1, 1, 1, device="cuda")
    return m, m * m + 0.5 + torch.rand(B, G, 1, 1, 1, device="cuda")


def _affine(Cc):
    return (1 + 0.1 * torch.randn(Cc, device="cuda")).half(), (0.1 * torch.randn(Cc, device="cuda")).half()


def test_groupnorm_sync_exchange_inside_async_step(arenas):
    """Mode 1 (sync_gn) in an asynchronous step: pub = e + 1, rd = e.  The exchange must read THIS step's bank (e + 1): bank
    e holds different, finite statistics."""
    torch.manual_seed(30)
    B, Cc, H, W, G, n, e = 2, 320, 8, 16, 32, 2, 5
    nb = B * G * 8
    arena = arenas(n, [nb], rank=0)
    w, b_ = _affine(Cc)
    x = (torch.randn(B, Cc, H, W, device="cuda") + 0.3).half().contiguous(memory_format=torch.channels_last)
    mine, peer = _moments(x, G), _fake_moments(B, G)
    stale = [_fake_moments(B, G, 3.0) for _ in range(n)]
    arena.slot(e + 1, 0, 1, nb, torch.float32).copy_(_pack(*peer).flatten())
    for s in range(n):
        arena.slot(e, 0, s, nb, torch.float32).copy_(_pack(*stale[s]).flatten())
    arena.flags[0, 0] = e
    arena.flags[0, 1] = e + 1
    arena.set_clock(pub=e + 1, rd=e)
    ref = _gn_ref(x, G, w, b_, 1e-5, (mine[0] + peer[0]) / 2, (mine[1] + peer[1]) / 2)
    wrong = _gn_ref(x, G, w, b_, 1e-5, (stale[0][0] + stale[1][0]) / 2, (stale[0][1] + stale[1][1]) / 2)
    assert (wrong - ref).abs().max().item() > 0.1, "bank e must hold statistics that change the output"
    y = _gn_call(x, G, w, b_, 1e-5, 1, 1, 0, 0, arena.comm, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b11)
    err = (y.float() - ref).abs().max().item()
    got = arena.slot(e + 1, 0, 0, nb, torch.float32).view(B * G, 2)
    assert err < 6e-3, f"max abs err {err}"
    assert (got - _pack(*mine)).abs().max().item() < 1e-4 and int(arena.flags[0, 0].item()) == e + 1


def test_groupnorm_corrected_negative_variance_fallback(arenas):
    """corrected_async_gn with neg_var_fallback: x_old scaled up in every third group makes the corrected variance negative
    there (checked in fp64 before the launch); exactly those groups must use the local variance."""
    torch.manual_seed(31)
    B, Cc, H, W, G, n, e = 2, 320, 8, 16, 32, 2, 5
    nb = B * G * 8
    arena = arenas(n, [nb], rank=0)
    w, b_ = _affine(Cc)
    x_now = (torch.randn(B, Cc, H, W, device="cuda") + 0.3).half().contiguous(memory_format=torch.channels_last)
    x_peer = (torch.randn(B, Cc, H, W, device="cuda") * 1.5).half()
    gscale = torch.ones(B, G, device="cuda")
    gscale[:, ::3] = 4.0
    x_old = ((torch.randn(B, Cc, H, W, device="cuda") * 0.7 - 0.2) * gscale.repeat_interleave(Cc // G, 1)[:, :, None, None]).half()
    mine, peer, old = (tuple(t.double() for t in _moments(x, G)) for x in (x_now, x_peer, x_old))
    mean = (old[0] + peer[0]) / 2 + (mine[0] - old[0])
    msq = (old[1] + peer[1]) / 2 + (mine[1] - old[1])
    var_c, var_local = msq - mean * mean, mine[1] - mine[0] ** 2
    neg = var_c < 0
    assert 0 < int(neg.sum()) < neg.numel() // 2, f"{int(neg.sum())} of {neg.numel()} groups negative"
    assert (var_c[neg] < -0.5).all() and (var_c[~neg] > 0.5).all(), "signs must be robust to fp32 rounding"
    assert ((var_c - var_local).abs()[~neg] > 0.1).all(), "the fallback must be visible in the groups that do not take it"
    arena.slot(e, 0, 1, nb, torch.float32).copy_(_pack(*peer).flatten())
    arena.slot(e, 0, 0, nb, torch.float32).copy_(_pack(*old).flatten())
    arena.flags[0, 0] = e
    arena.flags[0, 1] = e
    arena.set_clock(pub=e + 1, rd=e)
    y = _gn_call(x_now, G, w, b_, 1e-5, 2, 1, 1, 0, arena.comm, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b11)
    ref = _gn_ref(x_now, G, w, b_, 1e-5, mean, torch.where(neg, var_local + mean * mean, msq), bessel=True)
    err = (y.float() - ref).abs().max().item()
    assert torch.isfinite(y).all() and err < 6e-3, f"max abs err {err}"


@pytest.mark.parametrize("rank", [0, 1, 3])
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_groupnorm_halo_with_exchange(arenas, mode, rank):
    """df_groupnorm_halo_fwd at n=4 inside an asynchronous step (pub = e + 1, rd = e): statistics (tensor 0) and halo rows
    (tensor 1) in one arena.  Checks the normalised interior, the shipped rows (bank e + 1), the margins (bank e; the other
    bank of each neighbour poisoned), the published statistics and both flags."""
    torch.manual_seed(32 + 4 * mode + rank)
    b, c, h, w, G, n, e = 2, 64, 6, 10, 8, 4, 9
    pub, rd = e + 1, e
    up = rank - 1 if rank > 0 else -1
    down = rank + 1 if rank < n - 1 else -1
    nb, hb = b * G * 8, 2 * b * w * c * 2
    arena = arenas(n, [nb, hb], rank=rank)
    x = (torch.randn(b, c, h, w, device="cuda") * 2 + 0.3).half().contiguous(memory_format=torch.channels_last)
    gw, gb = _affine(c)
    mine = _moments(x, G)
    now = [_fake_moments(b, G) for _ in range(n)]            # the peers' statistics of this step (mode 1)
    old = [_fake_moments(b, G) for _ in range(n)]            # every member's statistics of the previous step (modes 2, 3)
    for s in range(n):
        arena.slot(rd, 0, s, nb, torch.float32).copy_(_pack(*old[s]).flatten())
        if s != rank:
            arena.slot(pub, 0, s, nb, torch.float32).copy_(_pack(*now[s]).flatten())
        arena.flags[0, s] = pub if (mode == 1 and s != rank) else rd
    top_src = torch.randn(b, w, c, device="cuda").half()
    bot_src = torch.randn(b, w, c, device="cuda").half()
    for nbr, part, src in ((up, 1, top_src), (down, 0, bot_src)):
        if nbr >= 0:
            arena.slot(rd, 1, nbr, hb).view(2, b, w, c)[part].copy_(src)
            arena.slot(pub, 1, nbr, hb).fill_(float("nan"))
            arena.flags[1, nbr] = rd
    arena.set_clock(pub=pub, rd=rd)
    if mode == 1:
        others = [now[s] for s in range(n) if s != rank]
        mean = (mine[0] + sum(o[0] for o in others)) / n
        msq = (mine[1] + sum(o[1] for o in others)) / n
    else:
        s0, s1 = sum(o[0] for o in old), sum(o[1] for o in old)
        if mode == 2:
            mean, msq = s0 / n + (mine[0] - old[rank][0]), s1 / n + (mine[1] - old[rank][1])
        else:
            mean, msq = (s0 - old[rank][0] + mine[0]) / n, (s1 - old[rank][1] + mine[1]) / n
    assert (msq - mean * mean).min().item() > 0.1, "the negative-variance fallback has its own test"
    yp = torch.full((b, c, h + 2, w), float("nan"), dtype=torch.float16, device="cuda").contiguous(memory_format=torch.channels_last)
    scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(b, G, h, w, c), dtype=torch.uint8, device="cuda")
    _check(_L().df_groupnorm_halo_fwd(arena.comm, x.data_ptr(), None, 0, yp.data_ptr(), gw.data_ptr(), gb.data_ptr(), b, h, w, c, G,
                                      1e-5, mode, 1, int(mode == 2), 1, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b1111,
                                      scratch.data_ptr(), 1, arena.tensor_off[1], arena.slot_bytes[1], up, down, 1, 1, _stream()),
           "df_groupnorm_halo_fwd")
    torch.cuda.synchronize()
    ref = _gn_ref(x, G, gw, gb, 1e-5, mean, msq, bessel=True, silu=True)
    ypn = yp.permute(0, 2, 3, 1)
    err = (ypn[:, 1:-1].float() - ref.permute(0, 2, 3, 1)).abs().max().item()
    assert err < 6e-3, f"max abs err {err}"
    assert torch.equal(ypn[:, 0], top_src if up >= 0 else torch.zeros_like(top_src)), "top margin"
    assert torch.equal(ypn[:, -1], bot_src if down >= 0 else torch.zeros_like(bot_src)), "bottom margin"
    shipped = arena.slot(pub, 1, rank, hb).view(2, b, w, c)
    if up >= 0:
        assert torch.equal(shipped[0], ypn[:, 1]), "first row shipped to the up neighbour"
    if down >= 0:
        assert torch.equal(shipped[1], ypn[:, h]), "last row shipped to the down neighbour"
    got = arena.slot(pub, 0, rank, nb, torch.float32).view(b * G, 2)
    assert (got - _pack(*mine)).abs().max().item() < 1e-4, "published statistics"
    assert int(arena.flags[0, rank].item()) == pub and int(arena.flags[1, rank].item()) == pub


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("B,Cc,H,W,G,halo,bessel", [
    pytest.param(2, 64, 1, 10, 8, True, 0, id="h1-halo"),            # one row: shipped up and down, both margins
    pytest.param(2, 256, 1, 1, 32, False, 0, id="hw1"),
    pytest.param(16, 64, 4, 4, 32, False, 0, id="bG512"),            # b * G at the exchange buffer's limit
    pytest.param(2, 256, 8, 8, 128, False, 0, id="G128"),
    pytest.param(1, 4096, 4, 6, 32, False, 0, id="C4096"),           # 512 channel vectors: one pixel lane per CTA
    pytest.param(2, 8, 16, 16, 8, False, 0, id="C8-G8"),             # one channel per group
    pytest.param(2, 320, 8, 8, 32, False, 1, id="bessel"),
])
def test_groupnorm_edge_shapes(arenas, mode, B, Cc, H, W, G, halo, bessel):
    """Local statistics (mode 0) and a synchronous exchange with two peers (mode 1, n=3, this rank in the middle)."""
    torch.manual_seed(33)
    n, rank, e = 3, 1, 4
    nb, hb = B * G * 8, 2 * B * W * Cc * 2
    arena = arenas(n, [nb, hb], rank=rank)
    x = (torch.randn(B, Cc, H, W, device="cuda") * 2 + 0.5).half().contiguous(memory_format=torch.channels_last)
    w, b_ = _affine(Cc)
    mean, msq = _moments(x, G)
    if mode == 1:
        for s in (0, 2):
            pm = _fake_moments(B, G)
            arena.slot(e, 0, s, nb, torch.float32).copy_(_pack(*pm).flatten())
            arena.flags[0, s] = e
            mean, msq = mean + pm[0], msq + pm[1]
        mean, msq = mean / n, msq / n
    arena.set_clock(pub=e, rd=e)
    ref = _gn_ref(x, G, w, b_, 1e-5, mean, msq, bessel=bool(bessel), silu=halo)
    if not halo:
        y = _gn_call(x, G, w, b_, 1e-5, mode, bessel, 0, 0, arena.comm, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b111)
        err = (y.float() - ref).abs().max().item()
        assert err < 6e-3, f"max abs err {err}"
        return
    assert H == 1
    top_src = torch.randn(B, W, Cc, device="cuda").half()
    bot_src = torch.randn(B, W, Cc, device="cuda").half()
    arena.slot(e, 1, 0, hb).view(2, B, W, Cc)[1].copy_(top_src)
    arena.slot(e, 1, 2, hb).view(2, B, W, Cc)[0].copy_(bot_src)
    arena.flags[1, 0] = e
    arena.flags[1, 2] = e
    yp = torch.full((B, Cc, H + 2, W), float("nan"), dtype=torch.float16, device="cuda").contiguous(memory_format=torch.channels_last)
    scratch = torch.zeros(_L().df_groupnorm_scratch_bytes(B, G, H, W, Cc), dtype=torch.uint8, device="cuda")
    _check(_L().df_groupnorm_halo_fwd(arena.comm, x.data_ptr(), None, 0, yp.data_ptr(), w.data_ptr(), b_.data_ptr(), B, H, W, Cc, G,
                                      1e-5, mode, bessel, 0, 1, 0, arena.tensor_off[0], arena.slot_bytes[0], 0b111,
                                      scratch.data_ptr(), 1, arena.tensor_off[1], arena.slot_bytes[1], 0, 2, 1, 1, _stream()),
           "df_groupnorm_halo_fwd")
    torch.cuda.synchronize()
    ypn = yp.permute(0, 2, 3, 1)
    err = (ypn[:, 1].float() - ref.permute(0, 2, 3, 1)[:, 0]).abs().max().item()
    assert err < 6e-3, f"max abs err {err}"
    shipped = arena.slot(e, 1, rank, hb).view(2, B, W, Cc)
    assert torch.equal(ypn[:, 0], top_src) and torch.equal(ypn[:, 2], bot_src), "margins"
    assert torch.equal(shipped[0], ypn[:, 1]) and torch.equal(shipped[1], ypn[:, 1]), "the one row goes up and down"
    assert int(arena.flags[1, rank].item()) == e


@pytest.mark.parametrize("offset", [8.0, 32.0])
def test_groupnorm_large_mean_offset(offset):
    """x = offset + N(0, 1): the variance is a small difference of large moments.  Against fp64 F.group_norm."""
    from distrifuser_b200 import _lib
    torch.manual_seed(34)
    B, Cc, H, W, G = 2, 320, 64, 64, 32
    x = (offset + torch.randn(B, Cc, H, W, device="cuda")).half().contiguous(memory_format=torch.channels_last)
    w, b_ = _affine(Cc)
    y = _gn_call(x, G, w, b_, 1e-5, 0, 0, 0, 0, _lib.null_comm(), 0, 0, 0, 1)
    ref = F.group_norm(x.double(), G, w.double(), b_.double(), 1e-5)
    err = (y.double() - ref).abs().max().item()
    print(f"groupnorm offset {offset}: max abs err {err:.3e}")
    assert err < 4e-3 * max(1.0, ref.abs().max().item() / 4), f"max abs err {err}"


# ================================================================================================================ output gather
@pytest.mark.parametrize("B,Cc,H,W,bs,me,vec", [
    pytest.param(1, 4, 16, 16, 1, 2, True, id="int4-row0"),
    pytest.param(1, 3, 12, 13, 1, 1, False, id="half-odd-width-row0"),
    pytest.param(2, 4, 8, 16, 1, 3, True, id="int4-batch0"),
    pytest.param(2, 3, 6, 13, 1, 3, False, id="half-batch0"),
])
def test_output_gather(arenas, B, Cc, H, W, bs, me, vec):
    """df_output_gather at n=4: the other ranks' strips sit in bank clock[2] (written by the test, flags stamped); this rank
    scatters its own strip at (batch0, row0) and collects the whole image bit-exactly.  The banks of clock[0] / clock[1]
    are poisoned."""
    n, E = 4, 11
    per = n // (B // bs)                                   # ranks per batch slice
    hs = H // per
    place = [((r // per) * bs, (r % per) * hs) for r in range(n)]
    assert ((hs * W) % 8 == 0) == vec and (place[me][0] > 0 or place[me][1] > 0)
    torch.manual_seed(35)
    img = torch.randn(B, Cc, H, W, device="cuda").half()
    nbytes = img.numel() * 2
    arena = arenas(n, [nbytes], rank=me)
    arena.set_clock(pub=E + 1, rd=E - 1)
    arena.clock[2] = E
    for ep in (E + 1, E - 1):
        arena.slot(ep, 0, 0, nbytes).fill_(float("nan"))
    bank = arena.slot(E, 0, 0, nbytes).view(B, Cc, H, W)
    for r in range(n):
        if r != me:
            b0, r0 = place[r]
            bank[b0:b0 + bs, :, r0:r0 + hs] = img[b0:b0 + bs, :, r0:r0 + hs]
            arena.flags[0, r] = E
    b0, r0 = place[me]
    strip = img[b0:b0 + bs, :, r0:r0 + hs].contiguous()
    out = torch.empty_like(img)
    _check(_L().df_output_gather(arena.comm, strip.data_ptr(), out.data_ptr(), B, Cc, H, W, bs, hs, b0, r0, 0,
                                 arena.tensor_off[0], _stream()), "df_output_gather")
    torch.cuda.synchronize()
    assert torch.equal(out, img)
    assert int(arena.flags[0, me].item()) == E


@pytest.mark.parametrize("kind,want", [(0, [6, 6, 10]), (1, [6, 5, 10]), (2, [5, 4, 10])])
def test_step_begin_clock(kind, want):
    """df_step_begin from (publish 5, read 4, output 9): synchronous, asynchronous, frozen."""
    clock = torch.tensor([5, 4, 9, 0], dtype=torch.int32, device="cuda")
    _check(_L().df_step_begin(clock.data_ptr(), kind, _stream()), "df_step_begin")
    torch.cuda.synchronize()
    assert clock.tolist() == want + [0]


# ================================================================================================================ GEMM
def _linear(a, w, out, bias=None, residual=None, epilogue=0, geglu_block=0, publish=None, max_ctas=0):
    """df_linear_fwd on 2-D operands with their own row pitches; publish = (comm, pub_col0, idx, peer_mask, tensor_off, slot_bytes)."""
    from distrifuser_b200 import _lib
    M, K = a.shape
    N = w.shape[0]
    comm, pub_col0, idx, mask, off, sb = publish if publish else (_lib.null_comm(), 0, 0, 0, 0, 0)
    _check(_L().df_linear_fwd(comm, a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                              residual.data_ptr() if residual is not None else None, out.data_ptr(), M, N, K, a.stride(0), w.stride(0),
                              residual.stride(0) if residual is not None else 0, out.stride(0), epilogue, geglu_block,
                              int(publish is not None), pub_col0, idx, mask, off, sb, max_ctas, _stream()), "df_linear_fwd")
    torch.cuda.synchronize()
    return out


def _tile_width(M, N, ctas):
    """pick_bn of csrc/linear.cu for the plain epilogue: 160-wide tiles where they cost < 0.97x the rounds x width of 256."""
    def cost(bn):
        return _cdiv(_cdiv(M, 128) * _cdiv(N, bn), ctas) * (bn + 64)
    return 160 if cost(160) < 0.97 * cost(256) else 256


def _operands(M, N, K, seed):
    torch.manual_seed(seed)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).half()
    return x, w


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("block", [80, 128])
def test_linear_geglu_forced_block(block, with_bias):
    """GEGLU with D = 1280: N = 2D tiles at both widths, so the caller may force either interleave block."""
    from distrifuser_b200 import ops
    M, K, D = 300, 320, 1280
    assert (2 * D) % 160 == 0 and (2 * D) % 256 == 0
    x, w = _operands(M, 2 * D, K, 40)
    b = (0.5 * torch.randn(2 * D, device="cuda")).half() if with_bias else None
    wi, bi = ops.geglu_interleave(w, b, block)
    out = _linear(x, wi, torch.empty(M, D, device="cuda", dtype=torch.float16), bias=bi, epilogue=1, geglu_block=block)
    y = x.float() @ w.float().t()
    if b is not None:
        y = y + b.float()
    y = y.half().float()
    _close(out, y[:, :D] * F.gelu(y[:, D:]), rel=4e-3, abs_=4e-3)


@pytest.mark.parametrize("max_ctas,bn", [(1, 256), (7, 256), (66, 160)])
def test_linear_max_ctas(max_ctas, bn):
    """CTA caps on a problem with row and column tails; the cap also moves the tile width (bn: the width pick_bn takes)."""
    M, N, K = 1000, 1000, 128
    assert M % 128 and N % 160 and N % 256 and _tile_width(M, N, max_ctas) == bn
    x, w = _operands(M, N, K, 41)
    b = torch.randn(N, device="cuda").half()
    out = _linear(x, w, torch.empty(M, N, device="cuda", dtype=torch.float16), bias=b, max_ctas=max_ctas)
    _close(out, x.float() @ w.float().t() + b.float())


def test_linear_output_and_residual_column_slices():
    """out and residual are column slices of wider buffers (ldo, ldr > N); the neighbouring columns stay untouched."""
    M, N, K = 300, 520, 192
    x, w = _operands(M, N, K, 42)
    b = torch.randn(N, device="cuda").half()
    r_wide = torch.randn(M, N + 24, device="cuda").half()
    r = r_wide[:, 8:8 + N]
    o_wide = torch.full((M, N + 40), 7.0, device="cuda", dtype=torch.float16)
    out = o_wide[:, 16:16 + N]
    assert out.stride(0) > N and r.stride(0) > N
    _linear(x, w, out, bias=b, residual=r)
    _close(out, (x.float() @ w.float().t() + b.float()).half().float() + r.float())
    assert (o_wide[:, :16] == 7).all() and (o_wide[:, 16 + N:] == 7).all(), "columns outside the output slice were written"


def test_linear_publish_with_bias_and_residual(arenas):
    """Publication of the columns >= pub_col0 (not on a tile boundary) with bias and residual and a row tail: the slot holds
    exactly the stored output columns, the flag carries the publish epoch."""
    M, N, K, pub_col0, me = 300, 640, 128, 200, 1
    assert pub_col0 % 160 and pub_col0 % 256 and M % 128
    x, w = _operands(M, N, K, 43)
    b = torch.randn(N, device="cuda").half()
    r = torch.randn(M, N, device="cuda").half()
    nbytes = M * (N - pub_col0) * 2
    arena = arenas(2, [nbytes], rank=me)
    arena.set_clock(pub=6, rd=5)
    out = _linear(x, w, torch.empty(M, N, device="cuda", dtype=torch.float16), bias=b, residual=r,
                  publish=(arena.comm, pub_col0, 0, 0b11, arena.tensor_off[0], arena.slot_bytes[0]))
    _close(out, (x.float() @ w.float().t() + b.float()).half().float() + r.float())
    assert torch.equal(arena.slot(6, 0, me, nbytes).view(M, N - pub_col0), out[:, pub_col0:])
    assert int(arena.flags[0, me].item()) == 6


def test_linear_minimal_shape():
    M, N, K = 1, 8, 64
    x, w = _operands(M, N, K, 44)
    b = torch.randn(N, device="cuda").half()
    r = torch.randn(M, N, device="cuda").half()
    out = _linear(x, w, torch.empty(M, N, device="cuda", dtype=torch.float16), bias=b, residual=r)
    _close(out, (x.float() @ w.float().t() + b.float()).half().float() + r.float())
