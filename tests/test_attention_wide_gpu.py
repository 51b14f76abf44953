"""GPU parity of the attention kernel for one head of width 512 (df_attn_wide_fwd, csrc/attention_wide.cu: the VAE decoder's
mid-block attention) against an fp32 torch restatement: one segment, and 2, 3 and 8 segments of unequal length whose peers'
parts are read in place from a loopback arena's slots (the next bank poisoned with NaN), as the ragged tests of df_attn_fwd do;
then the 230 400-token shape of a 3840 x 3840 image's 480 x 480 latent."""
import pytest
import torch

from helpers import LoopbackArena, _sdpa_ref_chunked

pytestmark = pytest.mark.gpu

D = 512


def _lib():
    from distrifuser_b200 import _lib
    return _lib


def wide_attn(q, segs, own, epoch=7, scale=0.0):
    """df_attn_wide_fwd with segs[own] as the own fresh segment, the others read from their arena slots."""
    _l = _lib()
    L = _l.lib()
    st = torch.cuda.current_stream().cuda_stream
    n, b = len(segs), q.shape[0]
    lens = [s.shape[1] for s in segs]
    arena, maps, comm = None, None, _l.null_comm()
    if n > 1:
        nbytes = [s.numel() * 2 for s in segs]
        arena = LoopbackArena(n, [max(nbytes)], rank=own)
        for s in range(n):
            if s != own:
                arena.slot(epoch, 0, s, nbytes[s]).copy_(segs[s].reshape(-1))
                arena.slot(epoch + 1, 0, s, max(nbytes)).fill_(float("nan"))
                arena.flags[0, s] = epoch
        arena.set_clock(pub=epoch + 1, rd=epoch)
        maps = torch.empty(_l.NBANKS * n * _l.TENSORMAP_BYTES, dtype=torch.uint8, device="cuda")
        _l.check(L.df_attn_wide_make_kvmaps(arena.comm, arena.tensor_off[0], arena.slot_bytes[0], b, _l.int32_array(lens), D,
                                            maps.data_ptr(), st), "df_attn_wide_make_kvmaps")
        comm = arena.comm
    out = torch.empty(q.shape, dtype=q.dtype, device="cuda")
    try:
        _l.check(L.df_attn_wide_fwd(comm, q.data_ptr(), segs[own].data_ptr(), out.data_ptr(),
                                    maps.data_ptr() if maps is not None else None, b, q.shape[1], _l.int32_array(lens), D,
                                    q.stride(1), segs[own].stride(1), out.stride(1), n, own, _l.int32_array(range(8)), 0, 1,
                                    scale, st), "df_attn_wide_fwd")
        torch.cuda.synchronize()
    finally:
        if arena is not None:
            arena.close()
    return out


def uneven(total, n, skew=37):
    """n segment lengths summing to `total`, all different when n > 1 (the first takes what the others give up)."""
    lens = [total // n + (1 if r < total % n else 0) for r in range(n)]
    for r in range(1, n):
        lens[r] -= skew * r % 61 + 1
        lens[0] += skew * r % 61 + 1
    assert sum(lens) == total and min(lens) >= 1
    return lens


def _check(out, ref):
    err = (out.float() - ref).abs().max().item()
    peak = ref.abs().max().item()
    assert err <= 2e-3 * peak, f"max |err| {err:.3e} > 2e-3 x max |ref| {peak:.3e}"
    assert torch.isfinite(out).all()


@pytest.mark.parametrize("nseg", [1, 2, 3, 8])
@pytest.mark.parametrize("L", [1024, 4097, 16384, 57600])
def test_wide_attention_segments(L, nseg):
    """Q = the own segment's rows (all L rows with one segment), K/V = all segments in rank order."""
    torch.manual_seed(L + nseg)
    lens = uneven(L, nseg)
    own = nseg // 2
    segs = [torch.randn(1, x, 2 * D, device="cuda", dtype=torch.float16) for x in lens]
    q = torch.randn(1, lens[own], D, device="cuda", dtype=torch.float16)
    out = wide_attn(q, segs, own)
    full = torch.cat([s.float() for s in segs], 1)
    _check(out, _sdpa_ref_chunked(q, full[..., :D], full[..., D:], 1, chunk=2048))


def test_wide_attention_batch_pitch_scale():
    """Two batch items, Q / K|V as column views of one fused q|k|v projection (row pitch 1536), an explicit scale."""
    torch.manual_seed(3)
    b, lens, own = 2, [1000, 777, 1300], 1
    segs = [torch.randn(b, x, 3 * D, device="cuda", dtype=torch.float16)[..., D:] for x in lens]
    segs = [s if i == own else s.contiguous() for i, s in enumerate(segs)]
    qkv = torch.randn(b, lens[own], 3 * D, device="cuda", dtype=torch.float16)
    q, segs[own] = qkv[..., :D], qkv[..., D:]
    out = wide_attn(q, segs, own, scale=0.03)
    full = torch.cat([s.float() for s in segs], 1)
    ref = _sdpa_ref_chunked(q * (0.03 * D ** 0.5), full[..., :D], full[..., D:], 1, chunk=2048)
    _check(out, ref)


def test_wide_attention_3840_world1():
    """The whole mid-block attention of a 3840 x 3840 image on one GPU: L = 480 * 480 = 230 400 tokens."""
    torch.manual_seed(0)
    L = 480 * 480
    kv = torch.randn(1, L, 2 * D, device="cuda", dtype=torch.float16)
    q = torch.randn(1, L, D, device="cuda", dtype=torch.float16)
    out = wide_attn(q, [kv], 0)
    rows = torch.arange(0, L, 97, device="cuda")                    # every 97th query row against the fp32 restatement
    _check(out[:, rows], _sdpa_ref_chunked(q[:, rows], kv[..., :D], kv[..., D:], 1, chunk=256))


def test_wide_attention_rejects_other_widths():
    _l = _lib()
    q = torch.zeros(1, 64, 256, device="cuda", dtype=torch.float16)
    kv = torch.zeros(1, 64, 512, device="cuda", dtype=torch.float16)
    rc = _l.lib().df_attn_wide_fwd(_l.null_comm(), q.data_ptr(), kv.data_ptr(), q.data_ptr(), None, 1, 64, _l.int32_array([64]),
                                   256, 256, 512, 256, 1, 0, _l.int32_array(range(8)), 0, 0, 0.0,
                                   torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"512" in _l.lib().df_last_error()
