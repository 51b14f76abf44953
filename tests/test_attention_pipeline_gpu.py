"""GPU parity of the attention kernel's software pipeline (fmha_fwd_kernel: S of slice i + 1 and P V of slice i in flight
together, O's rescale deferred until that P V retires), against the fp32 `sdpa_ref`.  Each case targets one state the
overlapped order has: its prologue and drain on items of 1, 2 and 3 K/V tiles, a reference move whose O rescale waits for
the previous slice's P V, back-to-back work items of different heads and batches handed out by the ticket scheduler, split
units, and the SDXL level-1 shape of the benchmark."""
import pytest
import torch

from helpers import _attn, _sdpa_ref_chunked, sdpa_ref

pytestmark = pytest.mark.gpu


def _inputs(b, lq, lk, heads, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Cq = heads * d
    q = torch.randn(b, lq, Cq, device="cuda", dtype=torch.float16, generator=g)
    kv = torch.randn(b, lk, 2 * Cq, device="cuda", dtype=torch.float16, generator=g)
    return q, kv


def _check(q, kv, heads, tol=2e-3, **kw):
    Cq = q.shape[-1]
    out = _attn(q, kv, heads, **kw)
    ref = sdpa_ref(q, kv[..., :Cq], kv[..., Cq:], heads)
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out).all() and err < tol, f"max abs err {err}"


@pytest.mark.parametrize("d", [64, 80, 160])
@pytest.mark.parametrize("lk", [128, 256, 300])   # T = 1, 2, 3 K/V tiles per item (the third one ragged)
def test_items_of_few_tiles(lk, d):
    q, kv = _inputs(2, 256, lk, 2, d, seed=lk + d)
    _check(q, kv, 2)


@pytest.mark.parametrize("d,jump", [(64, 128), (64, 256), (80, 64), (80, 192), (160, 128)])
def test_reference_move_under_previous_pv(d, jump):
    """K rows from `jump` on are scaled up, so the row maxima grow by far more than 2^8 on the slice that starts there: the
    exponent reference moves while the previous slice's P V is still accumulating into O (jump 64 / 192 at d = 80: the second
    64-wide slice of a tile)."""
    heads = 2
    q, kv = _inputs(1, 256, 384, heads, d, seed=d + jump)
    q *= 4
    kv[:, jump:, :heads * d] *= 30
    _check(q, kv, heads, tol=4e-3)


@pytest.mark.parametrize("d", [64, 80])
def test_dynamic_schedule_across_heads_and_batches(d):
    """444 (or 222) one- and two-tile work units on 132 CTAs through the ticket counter: every CTA runs several units of
    different (batch, head) back to back, each head on its own logit scale."""
    b, heads = 3, 37 if d == 64 else 18
    q, kv = _inputs(b, 512, 200, heads, d, seed=d)
    scale = torch.linspace(0.25, 3.0, heads, device="cuda").repeat_interleave(d).to(torch.float16)
    q *= scale
    _check(q, kv, heads, tol=4e-3)
    _check(q, kv, heads, tol=4e-3, no_ws=True)     # the same units through the static lists


@pytest.mark.parametrize("d", [64, 80])
def test_split_units_with_late_large_logits(d):
    """Tiny grid, long K/V: each unit is cut into K/V parts; the large logits sit in the last part only, so the merge
    weights differ by orders of magnitude and each part runs its own pipeline from its first tile."""
    heads = 4
    q, kv = _inputs(1, 256, 4096, heads, d, seed=7 + d)
    q *= 2
    kv[:, 3500:, :heads * d] *= 6
    _check(q, kv, heads, tol=4e-3)


def test_sdxl_level1_shape():
    """SDXL 1024^2 level-1 self-attention (2, 4096, 4096, 10 heads, d = 64): 640 units of 32 tiles on the dynamic schedule."""
    b, lq, heads, d = 2, 4096, 10, 64
    q, kv = _inputs(b, lq, lq, heads, d, seed=11)
    Cq = heads * d
    out = _attn(q, kv, heads)
    ref = _sdpa_ref_chunked(q, kv[..., :Cq], kv[..., Cq:], heads)
    err = (out.float() - ref).abs().max().item()
    assert err < 2e-3, f"max abs err {err}"
