"""GPU parity of the wgmma GEMM (csrc/linear.cu, df_linear_fwd) through the C ABI against fp32 torch restatements:
plain / bias / bias+residual epilogues, the fused GEGLU epilogue (diffusers GEGLU.forward) and the fused publication of
the k|v columns into the peers' arena slots.  Tolerance: fp16 storage of an fp32-accumulated result (|err| <= 2e-3 * |ref|
+ 2e-3 on O(1) data; K up to 5120)."""
import pytest
import torch

from helpers import LoopbackArena, _close

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [
    (256, 256, 64),            # one tile row pair, one K block
    (2048, 1280, 1280),        # SDXL level-2 attention projections at 1024^2 (to_out / to_q)
    (2048, 3840, 1280),        # fused q|k|v projection
    (8192, 640, 640),          # level 1: N = 2.5 tiles (column tail)
    (154, 2560, 2048),         # text K/V projection: 2 x 77 rows (row tail inside the second tile)
    (3600, 1280, 5120),        # 3840^2 n=4 level-2 FF2: ragged rows (3600 = 28 * 128 + 16), long K
    (300, 1288, 192),          # N % 8 == 0 only
])
@pytest.mark.parametrize("epi", ["plain", "bias", "bias_res"])
def test_linear_epilogues(M, N, K, epi):
    from distrifuser_b200 import ops
    torch.manual_seed(20)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).half()
    b = torch.randn(N, device="cuda").half() if epi != "plain" else None
    r = torch.randn(M, N, device="cuda").half() if epi == "bias_res" else None
    out = ops.linear(x, w, b, r)
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t()
    if b is not None:
        ref = ref + b.float()
    if r is not None:
        ref = ref.half().float() + r.float()        # torch: fp16 linear output, then fp16 add
    _close(out, ref)


def test_linear_strided_input_and_batched_shape():
    """A is a column slice of a wider matrix (pitch > K), 3-D input shape."""
    from distrifuser_b200 import ops
    torch.manual_seed(21)
    big = torch.randn(2, 700, 3 * 640, device="cuda").half()
    x = big[..., 640:1280]
    w = (torch.randn(1280, 640, device="cuda") / 25).half()
    out = ops.linear(x, w)
    ref = x.float() @ w.float().t()
    assert out.shape == (2, 700, 1280)
    _close(out, ref)


@pytest.mark.parametrize("M,K,D", [(2048, 1280, 5120), (8192, 640, 2560), (3600, 1280, 5120), (200, 320, 1280), (300, 64, 128), (500, 128, 80)])
def test_linear_geglu_fused(M, K, D):
    """diffusers GEGLU: y = proj(x); hidden, gate = y.chunk(2); hidden * gelu(gate) -- one kernel, interleaved weight."""
    from distrifuser_b200 import ops
    torch.manual_seed(22)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(2 * D, K, device="cuda") / K ** 0.5).half()
    b = (0.5 * torch.randn(2 * D, device="cuda")).half()
    block = ops.geglu_block(M, 2 * D, K)
    assert block in (80, 128)
    wi, bi = ops.geglu_interleave(w, b, block)
    out = ops.linear_geglu(x, wi, bi, block)
    torch.cuda.synchronize()
    y = (x.float() @ w.float().t() + b.float()).half().float()      # the projection is an fp16 tensor in diffusers
    ref = y[:, :D] * torch.nn.functional.gelu(y[:, D:])
    assert out.shape == (M, D)
    # one fp16 rounding of y before the gate (a 1-ulp flip of y moves the product by ~1e-3 relative) + one of the product
    _close(out, ref, rel=4e-3, abs_=4e-3)


def test_linear_repeated_launches_reuse_barriers():
    """Persistent CTAs and the smem ring (barrier phases) across many tiles and back-to-back launches."""
    from distrifuser_b200 import ops
    torch.manual_seed(23)
    x = torch.randn(4096, 640, device="cuda").half()
    w = (torch.randn(5120, 640, device="cuda") / 25).half()
    ref = x.float() @ w.float().t()
    for _ in range(3):
        out = ops.linear(x, w)
    torch.cuda.synchronize()
    _close(out, ref)


def test_linear_publishes_kv_columns_to_peer_slots():
    """Fused q|k|v projection: columns [C, 3C) land in slot(pub, idx, me) of every peer and the flag carries the epoch."""
    from distrifuser_b200 import ops
    torch.manual_seed(24)
    b, l, C, n, me = 2, 300, 640, 4, 1
    x = torch.randn(b, l, C, device="cuda").half()
    w = (torch.randn(3 * C, C, device="cuda") / 25).half()
    nbytes = b * l * 2 * C * 2
    arena = LoopbackArena(n, [nbytes, nbytes], rank=me)
    arena.set_clock(pub=6, rd=5)
    out = ops.linear(x, w, publish=(arena.comm, C, 1, 0b1101, arena.tensor_off[1], arena.slot_bytes[1]))
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t()
    _close(out, ref)
    got = arena.slot(6, 1, me, nbytes).view(b, l, 2 * C)
    flag = int(arena.flags[1, me].item())
    ok = torch.equal(got, out[..., C:])
    arena.close()
    assert ok and flag == 6
