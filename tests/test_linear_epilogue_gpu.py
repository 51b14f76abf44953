"""GPU tests of the GEMM's epilogue warps (csrc/linear.cu): the consumers stage each finished tile in shared memory and the
epilogue warps write it out while the next tile's mainloop runs.  Covers a staging buffer that wraps many times per CTA, back-to-back
launches of different shapes replayed from one CUDA graph, and the transformer-block Linears that ops.project routes to the GEMM."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from helpers import LoopbackArena, _close

pytestmark = pytest.mark.gpu


def _fwd(x, w, out, bias=None, residual=None, epilogue=0, geglu_block=0, publish=None, max_ctas=0):
    from distrifuser_b200 import _lib
    M, K = x.shape
    N = w.shape[0]
    comm, pub_col0, idx, mask, off, sb = publish if publish else (_lib.null_comm(), 0, 0, 0, 0, 0)
    _lib.check(_lib.lib().df_linear_fwd(comm, x.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                        residual.data_ptr() if residual is not None else None, out.data_ptr(), M, N, K,
                                        x.stride(0), w.stride(0), residual.stride(0) if residual is not None else 0,
                                        out.stride(0), epilogue, geglu_block, int(publish is not None), pub_col0, idx, mask,
                                        off, sb, max_ctas, torch.cuda.current_stream().cuda_stream), "df_linear_fwd")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
@pytest.mark.parametrize("epi", ["plain", "bias_res", "geglu80", "geglu128", "publish"])
def test_staging_wraps_over_many_tiles(epi, max_ctas):
    """M = 8192, N = 5120 on 1-3 CTAs: hundreds of tiles per CTA pass through the one staging buffer."""
    from distrifuser_b200 import ops
    M, N, K = (8120 if epi == "publish" else 8192), 5120, 128        # publish: a row tail in the last tile row
    torch.manual_seed(60)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).half()
    b = (0.5 * torch.randn(N, device="cuda")).half()
    if epi.startswith("geglu"):
        block, D = int(epi[5:]), N // 2
        wi, bi = ops.geglu_interleave(w, b, block)
        out = _fwd(x, wi, torch.empty(M, D, device="cuda", dtype=torch.float16), bias=bi, epilogue=1, geglu_block=block,
                   max_ctas=max_ctas)
        y = (x.float() @ w.float().t() + b.float()).half().float()
        _close(out, y[:, :D] * F.gelu(y[:, D:]), rel=4e-3, abs_=4e-3)
        return
    r = torch.randn(M, N, device="cuda").half()
    ref = (x.float() @ w.float().t() + b.float()).half().float() + r.float()
    if epi == "bias_res":
        _close(_fwd(x, w, torch.empty(M, N, device="cuda", dtype=torch.float16), bias=b, residual=r, max_ctas=max_ctas), ref)
        return
    pub_col0, me = 1680, 1                                           # not on a 256-column tile boundary
    nbytes = M * (N - pub_col0) * 2
    arena = LoopbackArena(2, [nbytes], rank=me)
    arena.set_clock(pub=6, rd=5)
    out = _fwd(x, w, torch.empty(M, N, device="cuda", dtype=torch.float16), bias=b, residual=r, max_ctas=max_ctas,
               publish=(arena.comm, pub_col0, 0, 0b11, arena.tensor_off[0], arena.slot_bytes[0]))
    got = arena.slot(6, 0, me, nbytes).view(M, N - pub_col0).clone()
    flag = int(arena.flags[0, me].item())
    arena.close()
    _close(out, ref)
    assert torch.equal(got, out[:, pub_col0:]) and flag == 6


def test_shapes_back_to_back_in_one_graph():
    """Plain, bias+residual and GEGLU launches of different shapes captured in one CUDA graph and replayed on new inputs."""
    from distrifuser_b200 import ops
    torch.manual_seed(61)
    x1, x2, x3 = (torch.empty(M, K, device="cuda").half() for M, K in [(2048, 1280), (8192, 640), (2048, 1280)])
    w1 = (torch.randn(1280, 1280, device="cuda") / 36).half()
    w2 = (torch.randn(640, 640, device="cuda") / 25).half()
    w3 = (torch.randn(10240, 1280, device="cuda") / 36).half()
    b1, b3 = torch.randn(1280, device="cuda").half(), (0.5 * torch.randn(10240, device="cuda")).half()
    r2 = torch.empty(8192, 640, device="cuda").half()
    block = ops.geglu_block(2048, 10240, 1280)
    w3i, b3i = ops.geglu_interleave(w3, b3, block)

    def run():
        return ops.linear(x1, w1, b1), ops.linear(x2, w2, None, r2), ops.linear_geglu(x3, w3i, b3i, block)

    for t in (x1, x2, x3, r2):
        t.normal_()
    run()                                            # eager first: kernel attributes are set outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = run()
    for _ in range(2):
        for t in (x1, x2, x3, r2):
            t.normal_()
        g.replay()
        torch.cuda.synchronize()
        _close(outs[0], x1.float() @ w1.float().t() + b1.float())
        _close(outs[1], (x2.float() @ w2.float().t()).half().float() + r2.float())
        y = (x3.float() @ w3.float().t() + b3.float()).half().float()
        _close(outs[2], y[:, :5120] * F.gelu(y[:, 5120:]), rel=4e-3, abs_=4e-3)


@pytest.fixture
def routed(monkeypatch):
    """Every kind on the hand-written GEMM; returns the list of (M, N, K) the GEMM ran."""
    from distrifuser_b200 import ops
    monkeypatch.setattr(ops, "_FUSED_LINEAR", {"geglu", "qkv", "out", "ff2", "proj"})
    calls = []
    real = ops.linear

    def spy(x, weight, *a, **kw):
        calls.append((x.numel() // x.shape[-1], weight.shape[0], x.shape[-1]))
        return real(x, weight, *a, **kw)

    monkeypatch.setattr(ops, "linear", spy)
    return calls


def _linear_module(cin, cout, bias=True, seed=0):
    torch.manual_seed(seed)
    lin = nn.Linear(cin, cout, bias=bias).cuda().half()
    with torch.no_grad():
        lin.weight.normal_(0, cin ** -0.5)
        if bias:
            lin.bias.normal_()
    return lin


@pytest.mark.parametrize("kind,M,cin,cout,bias", [
    ("out", 2048, 1280, 1280, True),      # attention to_out at level 2
    ("qkv", 2048, 1280, 1280, False),     # cross-attention to_q
    ("ff2", 8192, 2560, 640, True),       # FeedForward's second Linear at level 1
    ("proj", 2048, 1280, 1280, True),     # Transformer2DModel proj_in / proj_out (use_linear_projection)
])
def test_project_matches_linear(routed, kind, M, cin, cout, bias):
    from distrifuser_b200 import ops
    lin = _linear_module(cin, cout, bias, seed=62)
    x = torch.randn(2, M // 2, cin, device="cuda").half()
    out = ops.project(kind, x, lin)
    assert routed == [(M, cout, cin)]
    ref = x.float() @ lin.weight.float().t() + (lin.bias.float() if bias else 0)
    _close(out, ref)


def test_project_padded_to_out_weight(routed):
    """to_out of heads narrower than 64: the caller passes the zero-padded weight, the module's bias is used."""
    from distrifuser_b200 import ops
    lin = _linear_module(320, 320, seed=63)
    w_pad = F.pad(lin.weight.detach().reshape(320, 8, 40), (0, 24)).reshape(320, 512).contiguous()
    x = torch.randn(2, 4096, 512, device="cuda").half()
    out = ops.project("out", x, lin, w_pad)
    assert routed == [(8192, 320, 512)]
    _close(out, x.float() @ w_pad.float().t() + lin.bias.float())


def test_feedforward_routes_ff2(routed):
    """compat FeedForward: the fused GEGLU projection, then FF2 on the GEMM."""
    from distrifuser_b200.compat.unet_2d_condition import FeedForward
    torch.manual_seed(64)
    ff = FeedForward(640).cuda().half()
    x = torch.randn(2, 4096, 640, device="cuda").half()
    out = ff(x)
    assert (8192, 640, 2560) in routed
    p, lin2 = ff.net[0].proj, ff.net[2]
    y = (x.float() @ p.weight.float().t() + p.bias.float()).half().float()
    h = (y[..., :2560] * F.gelu(y[..., 2560:])).half().float()
    _close(out, h @ lin2.weight.float().t() + lin2.bias.float(), rel=4e-3, abs_=4e-3)
