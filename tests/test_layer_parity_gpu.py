"""Per-layer parity of the full-size SDXL and SD1.5 UNets at production resolutions against an fp64 reference.

One eager product UNet call per workload (world 1, CFG batch 2, built as tests/mp_product.py builds it).  Hooks on the
product capture the fp16 input and output of every ResnetBlock2D, Transformer2DModel, BasicTransformerBlock (through
`forward_chained`: input x + pending, output x' + pending'), self- and cross-attention wrapper, FeedForward, Downsample2D,
Upsample2D and of the whole UNet.  Inside the hook, before any later pass can touch the tensors, the module with the same
qualified name in the oracle's diffusers stub (same state-dict keys, same seeded weights rounded through fp16) runs on the
captured input twice:
  R  the stub module in fp64 on the GPU (moved to fp64 only while it runs; attention q-chunked),
  B  the stub module in fp16 on the GPU: torch's own kernels (cuBLAS, cuDNN, flash SDPA, eager GroupNorm).
With e = |X - R|_2 / |R|_2 and m = max|X - R| / rms(R) for X = P (the product) and X = B, an output passes when
  e_P <= f_e * e_B + 2^-11,   m_P <= f_m * m_B + 2^-9,   e_P < 2^-7
with per-type factors (f_e, f_m) in FACTORS.  B is what a library fp16 computation of the same operation reaches, so the
bar scales with the output and the operation: a systematic error of 2^-8 of the output fails it
(test_layer_parity_detects_injected_errors).  `pytest -s` prints every row and the worst ratios per type."""
from __future__ import annotations

import dataclasses
import gc
import math
import time

import pytest
import torch

from oracle import workloads as W

pytestmark = pytest.mark.gpu

E_FLOOR, M_FLOOR, E_ABS = 2.0 ** -11, 2.0 ** -9, 2.0 ** -7

# (f_e, f_m) per module type: about 1.5x the worst e_P / e_B and m_P / m_B measured over the workloads below in three runs on
# one H100 80GB HBM3 (700 W).  The worst ratios were 0.81 / 1.05 (ResnetBlock2D), 0.98 / 1.23 (Transformer2DModel),
# 1.00 / 1.52 (BasicTransformerBlock), 1.00 / 1.16 (attn1), 1.00 / 1.16 (attn2), 0.91 / 1.21 (FeedForward), 1.00 / 1.00
# (Downsample2D, Upsample2D) and 0.79 / 0.90 (UNet): the product is as close to fp64 as torch's fp16 kernels are.
FACTORS = {
    "ResnetBlock2D": (1.25, 1.6),
    "Transformer2DModel": (1.5, 1.85),
    "BasicTransformerBlock": (1.55, 2.3),
    "attn1": (1.55, 1.75),
    "attn2": (1.55, 1.75),
    "FeedForward": (1.4, 1.85),
    "Downsample2D": (1.55, 1.55),
    "Upsample2D": (1.55, 1.55),
    "UNet": (1.2, 1.35),
}

COUNTS = {
    "sdxl": dict(ResnetBlock2D=17, Transformer2DModel=11, BasicTransformerBlock=70, attn1=70, attn2=70, FeedForward=70,
                 Downsample2D=2, Upsample2D=2, UNet=1),
    "sd15": dict(ResnetBlock2D=22, Transformer2DModel=16, BasicTransformerBlock=16, attn1=16, attn2=16, FeedForward=16,
                 Downsample2D=3, Upsample2D=3, UNet=1),
}


@dataclasses.dataclass(frozen=True)
class Workload:
    name: str
    family: str
    hw: tuple                  # latent rows, columns
    only: tuple = ()           # qualified names checked with their checked descendants; () = every module and the UNet
    counts: tuple = ()         # expected checks per type of a subset

    def case(self):
        return W.RaggedCase(self.name, family=self.family, world_size=1, lat_h=self.hw[0], lat_w=self.hw[1], steps=1)


WORKLOADS = (
    Workload("sd15_512", "sd15", (64, 64)),            # padded d = 40 heads at level 0; d = 80 / 160
    Workload("sd15_768", "sd15", (96, 96)),            # level-0 L = 9216 at d = 40
    Workload("sdxl_1024", "sdxl", (128, 128)),         # bench.py's default
    Workload("sdxl_1216x832", "sdxl", (152, 104)),     # aspect bucket: level-1 L = 3952 = 30 * 128 + 112, level-2 L = 988
    Workload("sdxl_3840", "sdxl", (480, 480),          # bench.py's hires block: its largest launches
             only=("down_blocks.0.resnets.0",                          # GroupNorm over 230 400 pixels per sample
                   "up_blocks.2.resnets.0",                            # 960 concatenated channels at level 0
                   "down_blocks.1.attentions.0",                       # L = 57 600, GEGLU M = 115 200
                   "down_blocks.2.attentions.0.transformer_blocks.0"),  # L = 14 400
             counts=(("ResnetBlock2D", 2), ("Transformer2DModel", 1), ("BasicTransformerBlock", 3), ("attn1", 3),
                     ("attn2", 3), ("FeedForward", 3))),
)


# ------------------------------------------------------------------------------------------------ reference side
def _sdpa_fp64(q, k, v):
    """softmax(q k^T / sqrt(d)) v in fp64 on [b, heads, L, d], q rows in chunks: the [b, heads, lq, lk] scores never exist."""
    out = torch.empty_like(q)
    rows = max(1, (1 << 27) // (q.shape[0] * q.shape[1] * k.shape[2]))
    kt = k.transpose(-1, -2) * q.shape[-1] ** -0.5
    for r0 in range(0, q.shape[2], rows):
        out[:, :, r0:r0 + rows] = torch.softmax(q[:, :, r0:r0 + rows] @ kt, -1) @ v
    return out


def _chunked_attention(attn):
    """Instance forward of a stub Attention: the stub's own forward (flash SDPA) below fp64, its restatement with q-chunked
    attention in fp64."""
    plain = attn.forward

    def forward(hidden_states, encoder_hidden_states=None, **kw):
        if hidden_states.dtype != torch.float64:
            return plain(hidden_states, encoder_hidden_states, **kw)
        b = hidden_states.shape[0]
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        d = attn.inner_dim // attn.heads
        split = lambda t: t.view(b, -1, attn.heads, d).transpose(1, 2)
        o = _sdpa_fp64(split(attn.to_q(hidden_states)), split(attn.to_k(ctx)), split(attn.to_v(ctx)))
        return attn.to_out[0](o.transpose(1, 2).reshape(b, -1, attn.inner_dim))
    return forward


_STUB = {}


def _stub(family):
    """The oracle's diffusers-stub UNet of `family` with the product's seeded weights, fp16 on the GPU (one family at a time)."""
    if family not in _STUB:
        _STUB.clear()
        gc.collect()
        torch.cuda.empty_cache()
        from diffusers.models.attention_processor import Attention
        stub = W.make_unet(family, 0).to("cuda", torch.float16)
        for m in stub.modules():
            if isinstance(m, Attention):
                m.forward = _chunked_attention(m)
        _STUB[family] = stub
    return _STUB[family]


def _tensors(x, fn):
    if torch.is_tensor(x):
        return fn(x) if x.is_floating_point() else x
    if isinstance(x, (tuple, list)):
        return type(x)(_tensors(v, fn) for v in x)
    if isinstance(x, dict):
        return {k: _tensors(v, fn) for k, v in x.items()}
    return x


def _run_fp64(mod, args, kwargs, root):
    """mod(*args, **kwargs) in fp64.  The whole UNet goes to fp64 one top-level block at a time; fp16 -> fp64 -> fp16 is exact."""
    from torch import nn
    handles = []
    try:
        if root:
            def up(m, a):
                m.double()

            def down(m, a, o):
                m.half()
            for c in mod.children():
                for blk in (c if isinstance(c, nn.ModuleList) else [c]):
                    handles += [blk.register_forward_pre_hook(up), blk.register_forward_hook(down)]
        else:
            mod.double()
        return mod(*_tensors(args, torch.Tensor.double), **_tensors(kwargs, torch.Tensor.double))
    finally:
        for h in handles:
            h.remove()
        mod.half()


def _first(out):
    return out[0] if isinstance(out, (tuple, list)) else out


def _errors(x, r):
    """(e, m) of x against r, in fp64."""
    d = x.double() - r
    rn = r.norm().item()
    return d.norm().item() / rn, d.abs().max().item() / (rn / math.sqrt(r.numel()))


# ------------------------------------------------------------------------------------------------ product side
@dataclasses.dataclass
class Row:
    name: str
    kind: str
    shape: tuple
    eP: float
    mP: float
    eB: float
    mB: float

    @property
    def b_finite(self):
        return math.isfinite(self.eB) and math.isfinite(self.mB)

    @property
    def ratios(self):
        return (self.eP / self.eB, self.mP / self.mB) if self.b_finite else (math.nan, math.nan)

    def passes(self):
        if not self.b_finite:                       # no library baseline: the absolute bar alone
            return self.eP < E_ABS
        fe, fm = FACTORS[self.kind]
        return self.eP <= fe * self.eB + E_FLOOR and self.mP <= fm * self.mB + M_FLOOR and self.eP < E_ABS

    def __str__(self):
        re, rm = self.ratios
        return (f"{self.kind:21s} {self.name or '<unet>':56s} {str(list(self.shape)):22s} e_P {self.eP:.2e} e_B {self.eB:.2e} "
                f"({re:6.3f}x)  m_P {self.mP:.2e} m_B {self.mB:.2e} ({rm:6.3f}x){'' if self.passes() else '  FAIL'}")


class LayerParity:
    """Installs the capture hooks on a product UNet (the compat model inside DistriUNetPP) and collects one Row per checked
    output.  `tamper[name]` (tests only) rewrites that module's product output before it is compared and passed on."""

    def __init__(self, model, stub, only=()):
        from distrifuser_b200.compat import unet_2d_condition as compat
        from distrifuser_b200.modules.pp.attn import DistriCrossAttentionPP, DistriSelfAttentionPP
        self.stub, self.rows, self.tamper = stub, [], {}
        kinds = ((compat.ResnetBlock2D, "ResnetBlock2D"), (compat.Transformer2DModel, "Transformer2DModel"),
                 (compat.BasicTransformerBlock, "BasicTransformerBlock"), (DistriSelfAttentionPP, "attn1"),
                 (DistriCrossAttentionPP, "attn2"), (compat.FeedForward, "FeedForward"),
                 (compat.Downsample2D, "Downsample2D"), (compat.Upsample2D, "Upsample2D"))
        self.checked = {}
        for name, m in model.named_modules():
            if only and not any(name == o or name.startswith(o + ".") for o in only):
                continue
            kind = "UNet" if name == "" else next((k for cls, k in kinds if isinstance(m, cls)), None)
            if kind is None:
                continue
            self.checked[name] = kind
            if kind == "BasicTransformerBlock":
                m.forward_chained = self._chained(m.forward_chained, name)
            else:
                m.register_forward_hook(self._hook(name, kind), with_kwargs=True)

    def _hook(self, name, kind):
        def hook(mod, args, kwargs, out):
            p = _first(out)
            if name in self.tamper:
                p = self.tamper[name](p)
                out = (p,) if isinstance(out, tuple) else p
            self._compare(name, kind, args, kwargs, p)
            return out
        return hook

    def _chained(self, orig, name):
        def forward_chained(x, pending, encoder_hidden_states=None):
            xo, po = orig(x, pending, encoder_hidden_states)
            if name in self.tamper:
                xo, po = self.tamper[name](xo), self.tamper[name](po)
            xin = x if pending is None else x + pending
            self._compare(name, "BasicTransformerBlock", (xin,), dict(encoder_hidden_states=encoder_hidden_states), xo + po)
            return xo, po
        return forward_chained

    @torch.no_grad()
    def _compare(self, name, kind, args, kwargs, p):
        mod = self.stub if name == "" else self.stub.get_submodule(name)
        b = _first(mod(*args, **kwargs)).float()
        r = _first(_run_fp64(mod, args, kwargs, root=name == ""))
        assert r.shape == p.shape == b.shape, f"{name}: product {tuple(p.shape)}, stub {tuple(r.shape)}"
        eP, mP = _errors(p, r)
        eB, mB = _errors(b, r) if torch.isfinite(b).all() else (math.nan, math.nan)
        self.rows.append(Row(name, kind, tuple(p.shape), eP, mP, eB, mB))


def _product(wl):
    from mp_product import _pipeline
    case = wl.case()
    return _pipeline(case, False), W.unet_config(case.family)


def _call(pipe, ucfg, wl):
    """One eager UNet call on the case's first inputs, as tests/mp_product.py makes it."""
    model, dev = pipe.pipeline.unet, pipe.distri_config.device
    inp = W.unet_inputs(wl.case(), 0, ucfg)
    to_dev = lambda x: x.to(dev, torch.float16) if x.is_floating_point() else x.to(dev)
    kw = dict(sample=to_dev(inp["sample"]), timestep=inp["timestep"].to(dev).float(),
              encoder_hidden_states=to_dev(inp["encoder_hidden_states"]))
    if inp["added_cond_kwargs"] is not None:
        kw["added_cond_kwargs"] = {k: to_dev(v) for k, v in inp["added_cond_kwargs"].items()}
    with torch.no_grad():
        model.set_counter(0)
        out = model(**kw, return_dict=False)[0]
    torch.cuda.synchronize()
    return out


def _release():
    gc.collect()
    torch.cuda.empty_cache()


def _summary(rows):
    worst = {}
    for r in rows:
        re, rm = r.ratios
        we, wm, n = worst.get(r.kind, (0.0, 0.0, 0))
        worst[r.kind] = (max(we, re if math.isfinite(re) else 0.0), max(wm, rm if math.isfinite(rm) else 0.0), n + 1)
    return "\n".join(f"  {k:21s} n {n:3d}  worst e_P/e_B {we:6.3f}  worst m_P/m_B {wm:6.3f}" for k, (we, wm, n) in worst.items())


# ------------------------------------------------------------------------------------------------ tests
SD15_512 = WORKLOADS[0]

# one module of each checked type, none at a level too small for a 128-row tile (SD1.5, 64x64 latent)
TARGETS = {
    "down_blocks.0.resnets.1": "ResnetBlock2D",                                   # 320 channels, 64 x 64
    "down_blocks.1.attentions.0": "Transformer2DModel",                           # 640 channels, 1 024 tokens
    "up_blocks.3.attentions.2.transformer_blocks.0": "BasicTransformerBlock",     # 4 096 tokens
    "down_blocks.0.attentions.0.transformer_blocks.0.attn1": "attn1",             # d = 40, stored 64 wide
    "up_blocks.2.attentions.1.transformer_blocks.0.attn2": "attn2",               # d = 80
    "up_blocks.1.attentions.0.transformer_blocks.0.ff": "FeedForward",            # 1 280 channels, 256 tokens
    "down_blocks.1.downsamplers.0": "Downsample2D",                               # 640 channels, 16 x 16 out
    "up_blocks.2.upsamplers.0": "Upsample2D",                                     # 640 channels, 64 x 64 out
    "": "UNet",
}


def _scale_all(t):
    return t * (1 + 2.0 ** -8)


def _scale_tile(kind):
    """One 128-row x 64-column tile scaled by 1 + 2^-5: 128 tokens x 64 channels, or 128 pixels of one GroupNorm group's
    channels (ResnetBlock2D; all 4 channels of the UNet output)."""
    def fn(t):
        t = t.clone()
        if t.ndim == 3:
            t[0, 128:256, 64:128] *= 1 + 2.0 ** -5
        else:
            c = t.shape[1]
            c0, k = {"ResnetBlock2D": (c // 32, c // 32), "UNet": (0, c)}.get(kind, (64, 64))
            t.flatten(2)[0, c0:c0 + k, 128:256] *= 1 + 2.0 ** -5
        return t
    return fn


def _tile_in_attention(wrapper):
    """The attention kernel's output of one 128-row q tile of one head (rows 128..255, head 1) scaled by 1 + 2^-5."""
    attend = wrapper._attend

    def fn(q, *a, **k):
        out = attend(q, *a, **k).clone()
        d = q.shape[-1] // wrapper.module.heads
        out[0, 128:256, d:2 * d] *= 1 + 2.0 ** -5
        return out
    wrapper._attend = fn


def test_layer_parity_detects_injected_errors():
    """The bar rejects a module whose output is off by 2^-8 of its scale, or by 2^-5 on one 128 x 64 tile, and accepts every
    other module -- also those downstream of the error, which are checked on the input the product actually fed them.  The
    checked ancestors of a tampered module carry its error diluted by the rest of their output and are not asserted on."""
    stub = _stub(SD15_512.family)
    for label in ("scale 1 + 2^-8", "tile 1 + 2^-5"):
        pipe, ucfg = _product(SD15_512)
        model = pipe.pipeline.unet.model
        lp = LayerParity(model, stub)
        for name, kind in TARGETS.items():
            assert lp.checked[name] == kind
            if label.startswith("scale"):
                lp.tamper[name] = _scale_all
            elif kind in ("attn1", "attn2"):
                _tile_in_attention(model.get_submodule(name))
            else:
                lp.tamper[name] = _scale_tile(kind)
        _call(pipe, ucfg, SD15_512)
        ancestors = {n for n in lp.checked for t in TARGETS if n not in TARGETS and (n == "" or t.startswith(n + "."))}
        print(f"\n{label}:")
        for r in lp.rows:
            if r.name in TARGETS:
                print(f"  tampered {r}")
        missed = [str(r) for r in lp.rows if r.name in TARGETS and r.passes()]
        false = [str(r) for r in lp.rows if r.name not in TARGETS and r.name not in ancestors and not r.passes()]
        assert not missed, f"{label}: tampered modules accepted:\n" + "\n".join(missed)
        assert not false, f"{label}: untampered modules rejected:\n" + "\n".join(false)
        del pipe, model, lp
        _release()


@pytest.mark.parametrize("wl", WORKLOADS, ids=[w.name for w in WORKLOADS])
def test_layer_parity_vs_fp64(wl):
    stub = _stub(wl.family)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    pipe, ucfg = _product(wl)
    lp = LayerParity(pipe.pipeline.unet.model, stub, wl.only)
    _call(pipe, ucfg, wl)
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"\n{wl.name}: latent {wl.hw[0]}x{wl.hw[1]}, {len(lp.rows)} outputs checked, {wall:.0f} s, peak {peak:.1f} GiB allocated")
    for r in lp.rows:
        print(f"  {r}")
    print(_summary(lp.rows))
    no_b = [str(r) for r in lp.rows if not r.b_finite]
    if no_b:
        print("  library fp16 baseline not finite (absolute bar only):\n  " + "\n  ".join(no_b))
    counts = {}
    for r in lp.rows:
        counts[r.kind] = counts.get(r.kind, 0) + 1
    assert counts == (dict(wl.counts) if wl.only else COUNTS[wl.family]), f"{wl.name}: checked {counts}"
    bad = [str(r) for r in lp.rows if not r.passes()]
    del pipe, lp
    _release()
    assert not bad, f"{wl.name}: {len(bad)} outputs off the fp64 reference beyond the bar:\n" + "\n".join(bad)
