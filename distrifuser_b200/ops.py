"""Small fused ops on the per-step path that are not reference wrappers (thin shims over the C ABI)."""
import os as _os

import torch

from . import _lib


def geglu(y: torch.Tensor) -> torch.Tensor:
    """hidden * gelu_erf(gate) for y = [..., 2*cols] = [hidden | gate] (diffusers GEGLU.forward after the projection)."""
    assert y.is_cuda and y.dtype == torch.float16 and y.stride(-1) == 1
    cols = y.shape[-1] // 2
    y2 = y.reshape(-1, 2 * cols)
    out = torch.empty((*y.shape[:-1], cols), dtype=y.dtype, device=y.device)
    _lib.check(_lib.lib().df_geglu(y2.data_ptr(), out.data_ptr(), y2.shape[0], cols, y2.stride(0), cols,
                                   torch.cuda.current_stream().cuda_stream), "df_geglu")
    return out


def add_layernorm(x: torch.Tensor, r: torch.Tensor | None, norm: torch.nn.LayerNorm):
    """-> (x + r, LayerNorm(x + r)) in one kernel (r=None: (x, LayerNorm(x)))."""
    assert x.is_cuda and x.dtype == torch.float16
    C = x.shape[-1]
    x = x.contiguous()
    y = torch.empty_like(x)
    if r is not None:
        r = r.contiguous()
        s = torch.empty_like(x)
    else:
        s = x
    _lib.check(_lib.lib().df_add_layernorm(x.data_ptr(), r.data_ptr() if r is not None else None,
                                           s.data_ptr() if r is not None else None, y.data_ptr(), norm.weight.data_ptr(),
                                           norm.bias.data_ptr(), x.numel() // C, C, float(norm.eps),
                                           torch.cuda.current_stream().cuda_stream), "df_add_layernorm")
    return s, y


def conv2d_bias_residual(x: torch.Tensor, conv: torch.nn.Conv2d, padding, residual: torch.Tensor | None = None,
                         bias: torch.Tensor | None = None, fold_bias: bool = False) -> torch.Tensor:
    """conv(x) + bias (+ residual): the convolution runs in cuDNN WITHOUT bias and one vectorised pass adds `bias` (default
    conv.bias) and the residual (df_bias_residual_add).  fold_bias: the caller adds the bias elsewhere (e.g. into the addend of
    the following GroupNorm) -- no pass at all.  Falls back to F.conv2d for anything but fp16 CUDA NHWC tensors."""
    import torch.nn.functional as F
    b = conv.bias if bias is None else bias
    ok = (x.is_cuda and x.dtype == torch.float16 and conv.out_channels % 8 == 0 and
          x.is_contiguous(memory_format=torch.channels_last))
    if not ok:
        out = F.conv2d(x, conv.weight, None if fold_bias else b, stride=conv.stride, padding=padding)
        return out if residual is None else residual + out
    out = F.conv2d(x, conv.weight, None, stride=conv.stride, padding=padding)
    if (b is None or fold_bias) and residual is None:
        return out
    if not out.is_contiguous(memory_format=torch.channels_last):
        out = out.contiguous(memory_format=torch.channels_last)
    if b is None or fold_bias:
        return residual + out
    if residual is not None:
        assert residual.shape == out.shape and residual.dtype == out.dtype
        if not residual.is_contiguous(memory_format=torch.channels_last):
            residual = residual.contiguous(memory_format=torch.channels_last)
    n, c, h, w = out.shape
    _lib.check(_lib.lib().df_bias_residual_add(out.data_ptr(), residual.data_ptr() if residual is not None else None,
                                               b.data_ptr(), out.data_ptr(), n * h * w, c,
                                               torch.cuda.current_stream().cuda_stream), "df_bias_residual_add")
    return out


# ---------------------------------------------------------------------------------------------------- wgmma GEMM (csrc/linear.cu)

# which Linear layers run on the hand-written GEMM: comma list out of {geglu, qkv, out, ff2, proj}; "all" / "none".
# Default: the GEGLU projection, whose fused epilogue saves the [M, 8C] intermediate.  The plain kinds are slower than cuBLAS at
# the model's step shapes on H100 (tools/bench_linear.py, DESIGN §7), so they stay off by default.
_FUSED_LINEAR = set(_os.environ.get("DF_LINEAR", "geglu").replace("all", "geglu,qkv,out,ff2,proj").split(","))


def use_fused_linear(kind: str) -> bool:
    return kind in _FUSED_LINEAR


GEGLU_BLOCK = 128      # default rows of the interleaved GEGLU weight: [hidden block t | gate block t]; see geglu_block()


def linear_supported(M: int, N: int, K: int, geglu: bool = False) -> bool:
    return bool(_lib.lib().df_linear_supported(M, N, K, 1 if geglu else 0))


def geglu_block(M: int, two_d: int, K: int) -> int:
    """Rows per hidden / gate block the fused kernel wants for this problem (80 or 128; 0 = not supported): half of the tile
    width, chosen so that the tiles fill the SMs (160-wide tiles where they need clearly fewer rounds than 256-wide ones)."""
    if not linear_supported(M, two_d, K, geglu=True):
        return 0
    return int(_lib.lib().df_linear_geglu_block(M, two_d, K))


def geglu_interleave(weight: torch.Tensor, bias: torch.Tensor | None, block: int = GEGLU_BLOCK):
    """diffusers GEGLU.proj holds [hidden (D rows) ; gate (D rows)]; the fused kernel wants them interleaved in blocks of `block`
    rows so that one accumulator tile carries both halves of `block` outputs."""
    two_d, K = weight.shape
    D = two_d // 2
    assert D % block == 0
    w = torch.stack([weight[:D].reshape(D // block, block, K), weight[D:].reshape(D // block, block, K)], 1)
    w = w.reshape(two_d, K).contiguous()
    b = None
    if bias is not None:
        b = torch.stack([bias[:D].reshape(-1, block), bias[D:].reshape(-1, block)], 1).reshape(two_d).contiguous()
    return w, b


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None, residual: torch.Tensor | None = None,
           out: torch.Tensor | None = None, publish=None) -> torch.Tensor:
    """x[..., K] @ weight[N, K]^T (+ bias) (+ residual) on the hand-written wgmma GEMM.  `publish` = (comm, pub_col0, idx,
    peer_mask, tensor_off, slot_bytes): the columns >= pub_col0 also go into the peers' arena slots."""
    assert x.is_cuda and x.dtype == torch.float16 and weight.dtype == torch.float16 and x.stride(-1) == 1 and weight.stride(-1) == 1
    K = x.shape[-1]
    N = weight.shape[0]
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    if out is None:
        out = torch.empty((*x.shape[:-1], N), dtype=x.dtype, device=x.device)
    o2 = out.view(-1, N)
    r2 = residual.reshape(-1, N) if residual is not None else None
    if publish is not None:
        comm, pub_col0, idx, mask, off, sb = publish
    else:
        comm, pub_col0, idx, mask, off, sb = _lib.null_comm(), 0, 0, 0, 0, 0
    _lib.check(_lib.lib().df_linear_fwd(comm, x2.data_ptr(), weight.data_ptr(), bias.data_ptr() if bias is not None else None,
                                        r2.data_ptr() if r2 is not None else None, o2.data_ptr(), M, N, K, x2.stride(0),
                                        weight.stride(0), r2.stride(0) if r2 is not None else 0, o2.stride(0), 0, 0,
                                        int(publish is not None), pub_col0, idx, mask, off, sb, 0,
                                        torch.cuda.current_stream().cuda_stream), "df_linear_fwd")
    return out


def project(kind: str, x: torch.Tensor, lin: torch.nn.Linear, weight: torch.Tensor | None = None) -> torch.Tensor:
    """lin(x) for a transformer-block Linear of `kind` ("qkv", "out", "ff2", "proj"): on the hand-written GEMM when DF_LINEAR
    selects the kind, else lin itself (cuBLAS).  `weight` replaces lin.weight (zero-padded to_out of narrow heads).  A Linear
    with a LoRA layer attached keeps its own forward."""
    w = lin.weight if weight is None else weight
    K = x.shape[-1]
    if (use_fused_linear(kind) and x.is_cuda and x.dtype == torch.float16 and w.dtype == torch.float16 and
            x.stride(-1) == 1 and w.stride(-1) == 1 and getattr(lin, "lora_layer", None) is None and
            linear_supported(x.numel() // K, w.shape[0], K)):
        return linear(x, w, lin.bias)
    if weight is None:
        return lin(x)
    import torch.nn.functional as F
    return F.linear(x, weight, lin.bias)


def linear_geglu(x: torch.Tensor, w_interleaved: torch.Tensor, b_interleaved: torch.Tensor | None, block: int = GEGLU_BLOCK) -> torch.Tensor:
    """hidden * gelu_erf(gate) of the GEGLU projection in ONE kernel; weights from geglu_interleave(..., block)."""
    assert x.is_cuda and x.dtype == torch.float16 and x.stride(-1) == 1
    K = x.shape[-1]
    N = w_interleaved.shape[0]
    x2 = x.reshape(-1, K)
    out = torch.empty((*x.shape[:-1], N // 2), dtype=x.dtype, device=x.device)
    _lib.check(_lib.lib().df_linear_fwd(_lib.null_comm(), x2.data_ptr(), w_interleaved.data_ptr(),
                                        b_interleaved.data_ptr() if b_interleaved is not None else None, None, out.data_ptr(),
                                        x2.shape[0], N, K, x2.stride(0), w_interleaved.stride(0), 0, N // 2, 1, block, 0, 0, 0, 0, 0, 0, 0,
                                        torch.cuda.current_stream().cuda_stream), "df_linear_fwd")
    return out


def controlnet_zero_convs(xs, convs, scale: torch.Tensor) -> list[torch.Tensor]:
    """[scale * conv_i(xs[i]) for every 1x1 zero conv of a ControlNet call] in ONE launch (df_controlnet_zero_convs).  xs: fp16
    NHWC activations; convs: the nn.Conv2d 1x1 modules; scale: a device fp32 tensor of one element, read by the kernel."""
    import ctypes as C
    n = len(xs)
    assert len(convs) == n and scale.is_cuda and scale.dtype == torch.float32 and scale.numel() == 1
    outs, xp, wp, bp, op, ms, ns, ks = [], [], [], [], [], [], [], []
    for x, conv in zip(xs, convs):
        assert x.is_cuda and x.dtype == torch.float16 and tuple(conv.kernel_size) == (1, 1)
        x = x.contiguous(memory_format=torch.channels_last)
        b, k, h, w = x.shape
        out = torch.empty((b, conv.out_channels, h, w), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        outs.append(out)
        xp.append(x.data_ptr()); wp.append(conv.weight.data_ptr()); op.append(out.data_ptr())
        bp.append(conv.bias.data_ptr() if conv.bias is not None else None)
        ms.append(b * h * w); ns.append(conv.out_channels); ks.append(k)
    ptrs = lambda v: (C.c_void_p * n)(*v)
    _lib.check(_lib.lib().df_controlnet_zero_convs(n, ptrs(xp), ptrs(wp), ptrs(bp), ptrs(op), (C.c_int64 * n)(*ms),
                                                   (C.c_int32 * n)(*ns), (C.c_int32 * n)(*ks), scale.data_ptr(), 0,
                                                   torch.cuda.current_stream().cuda_stream), "df_controlnet_zero_convs")
    return outs
