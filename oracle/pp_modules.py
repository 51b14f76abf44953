"""TEST INFRASTRUCTURE (oracle) -- never imported by the product package.

CPU (torch fp32) restatement of the reference's patch-parallel hot path, written from its observable
behaviour, each piece citing the reference file:line it follows:

  * OracleComm            <- distrifuser/utils.py:112-199   (PatchParallelismCommManager)
  * OracleGroupNorm       <- distrifuser/modules/pp/groupnorm.py:14-97
  * OracleConv2d          <- distrifuser/modules/pp/conv2d.py:20-115
  * OracleSelfAttention   <- distrifuser/modules/pp/attn.py:107-195
  * OracleCrossAttention  <- distrifuser/modules/pp/attn.py:42-104
  * OracleUNetPP          <- distrifuser/models/distri_sdxl_unet_pp.py:16-210 (eager path)

Uneven row strips.  The reference asserts equal strips; these modules also restate the product's rule for a patch count
that does not divide the latent rows (distrifuser_b200.utils.split_units, restated here so that the check stays
independent): patch rank r of n holds `units[r]` units of 2^downsamplers latent rows, U // n each and one more for the
first U % n ranks.  K/V slots then hold segments of unequal length, every GroupNorm mean over ranks weighs rank s by
rows_s / sum(rows), and the conv_in slice and the final gather sit at the prefix sums of the rows.  Equal strips take the
reference's expressions unchanged.  `bessel=False` drops the local-count Bessel factor, so that an uneven full_sync run
equals the one-device UNet exactly.

PINNING: this restatement is checked against outputs of the UNMODIFIED reference modules executed in the
build container (oracle/make_golden.py imports them from /root/reference through oracle/diffusers_stub and
runs them under gloo); the resulting vectors are committed in tests/golden/ and compared in
tests/test_oracle_vs_golden.py.  The reference itself ships no tests or golden vectors (SURVEY 4), and the
diffusers-0.24.0 UNet topology around the modules is "parity unpinned" (see oracle/diffusers_stub).

Staleness model.  The reference ships activations with batched async all_gathers every `comm_checkpoint`
tensors and flushes the tail at the next step's first enqueue (utils.py:170-190).  For every registered
tensor count >= comm_checkpoint (SDXL 155/109, SD1.x 128; SURVEY D-13) the observable effect is: in an
asynchronous step every module reads exactly the values its peers produced ONE step earlier.  OracleComm
implements that contract directly (publish now, becomes visible at the next step's `begin_step`).
"""
from __future__ import annotations

import torch
from torch import distributed as dist
from torch import nn
from torch.nn import functional as F


# ----------------------------------------------------------------------------------------------- comm
def _all_gather_padded(local: torch.Tensor, sizes: list[int], dim: int, group) -> list[torch.Tensor]:
    """all_gather of tensors whose length along `dim` differs between the members (`sizes`): padded to the longest."""
    shape = list(local.shape)
    shape[dim] = max(sizes)
    padded = local.new_zeros(shape)
    padded.narrow(dim, 0, local.shape[dim]).copy_(local)
    bufs = [torch.empty_like(padded) for _ in sizes]
    dist.all_gather(bufs, padded, group=group)
    return [b.narrow(dim, 0, sz).contiguous() for b, sz in zip(bufs, sizes)]


class OracleComm:
    """Per-tensor peer slots with 1-step-stale visibility (utils.py:112-199)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.shapes: list[list[tuple]] = []                # per tensor, the shape of each source's slot
        self.slots: list[list[torch.Tensor]] | None = None
        self.pending: dict[int, torch.Tensor] = {}

    @property
    def n(self):
        return self.cfg.n_device_per_batch

    def register(self, shape, lens=None) -> int:           # utils.py:130-149
        """`lens`: each source's length along dim 1 (K/V of uneven strips); default: every source holds `shape`."""
        shape = tuple(shape)
        self.shapes.append([shape] * self.n if lens is None else [(shape[0], L, *shape[2:]) for L in lens])
        return len(self.shapes) - 1

    def create(self, dtype=torch.float32):                 # utils.py:151-164
        self.slots = [[torch.zeros(s, dtype=dtype) for s in shapes] for shapes in self.shapes]

    def _all_gather(self, idx: int, local: torch.Tensor):
        shapes = self.shapes[idx]
        if len(set(shapes)) == 1:
            dist.all_gather(self.slots[idx], local, group=self.cfg.batch_group)
        else:
            self.slots[idx] = _all_gather_padded(local, [s[1] for s in shapes], 1, self.cfg.batch_group)

    def gather_now(self, idx: int, local: torch.Tensor):
        """Blocking all_gather of a synchronous step (attn.py:133, conv2d.py:93, groupnorm.py:46)."""
        self._all_gather(idx, local.contiguous())
        return self.slots[idx]

    def publish(self, idx: int, local: torch.Tensor):      # utils.py:181-190 (enqueue)
        self.pending[idx] = local.detach().clone().contiguous()

    def begin_step(self):
        """Make everything published during the previous step visible (utils.py:170-179,183-184)."""
        for idx in sorted(self.pending):
            self._all_gather(idx, self.pending[idx])
        self.pending = {}


class _Wrapped(nn.Module):                                 # modules/base_module.py:6-29
    units: list[int] | None = None                         # row plan, set by OracleUNetPP (None: equal strips)
    bessel: bool = True

    def __init__(self, module, cfg):
        super().__init__()
        self.module, self.cfg = module, cfg
        self.comm: OracleComm | None = None
        self.counter = 0
        self.idx = None

    def set_counter(self, c=0):
        self.counter = c

    def set_comm(self, comm):
        self.comm = comm

    def _is_sync(self):                                    # attn.py:132 / conv2d.py:92 / groupnorm.py:45
        return self.counter <= self.cfg.warmup_steps

    def _bound(self):
        return self.comm is not None and self.comm.slots is not None and self.idx is not None

    def rows(self, h):
        """Rows of every patch rank where this rank holds h rows (tokens alike): distrifuser_b200.utils.patch_rows."""
        units = self.units or [1] * self.cfg.n_device_per_batch
        return [u * h // units[self.cfg.split_idx()] for u in units]

    def row_weights(self, h):
        """Each patch rank's share of the rows for uneven strips; None for equal strips (the reference's 1/n)."""
        if self.units is None or len(set(self.units)) == 1:
            return None
        rows = self.rows(h)
        return [s / sum(rows) for s in rows]


# ----------------------------------------------------------------------------------------------- GroupNorm
def _moments(x5):
    return torch.stack([x5.mean(dim=[2, 3, 4], keepdim=True), (x5 * x5).mean(dim=[2, 3, 4], keepdim=True)], 0)


class OracleGroupNorm(_Wrapped):
    def forward(self, x):
        m, cfg = self.module, self.cfg
        b, c, h, w = x.shape
        G = m.num_groups
        stat_modes = cfg.mode in ("stale_gn", "corrected_async_gn")
        if stat_modes and self.comm is not None and self.idx is None and self.comm.slots is None:
            self.idx = self.comm.register((2, b, G, 1, 1, 1))                       # groupnorm.py:29-35
        if not stat_modes and not (self._is_sync() or cfg.mode in ("sync_gn", "full_sync")):
            self.counter += 1
            return m(x)                                                             # groupnorm.py:92-93
        x5 = x.reshape(b, G, c // G, h, w)
        mine = _moments(x5)                                                         # groupnorm.py:38-41 / 75-78
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        wts = self.row_weights(h)
        avg = (lambda parts: sum(parts) / n) if wts is None else (lambda parts: sum(wt * g for wt, g in zip(wts, parts)))
        use_local_fallback = False
        if stat_modes:
            if not self._bound():
                full = mine                                                         # groupnorm.py:43-44
            elif self._is_sync():
                full = avg(self.comm.gather_now(self.idx, mine))                    # groupnorm.py:45-47
            else:
                stale = self.comm.slots[self.idx]
                if cfg.mode == "corrected_async_gn":                                # groupnorm.py:49-51
                    full = avg(stale) + (mine - stale[r])
                    use_local_fallback = True
                elif wts is None:                                                   # groupnorm.py:52-55
                    full = (sum(stale) - stale[r] + mine) / n
                else:
                    full = avg([mine if s == r else g for s, g in enumerate(stale)])
                self.comm.publish(self.idx, mine)                                   # groupnorm.py:56
            if cfg.mode == "corrected_async_gn":
                use_local_fallback = True                                           # groupnorm.py:60-63 (all steps)
        elif wts is None:                                                           # groupnorm.py:74-80
            full = mine.clone()
            if n > 1:
                dist.all_reduce(full, op=dist.ReduceOp.SUM, group=cfg.batch_group)
            full = full / n
        else:
            full = mine * wts[r]
            dist.all_reduce(full, op=dist.ReduceOp.SUM, group=cfg.batch_group)
        mean, meansq = full[0], full[1]
        var = meansq - mean * mean
        if use_local_fallback:
            var = torch.where(var < 0, mine[1] - mine[0] * mine[0], var)
        ne = (c // G) * h * w
        if self.bessel:
            var = var * (ne / (ne - 1))                                             # groupnorm.py:65-66,84-85
        y = ((x5 - mean) / (var + m.eps).sqrt()).reshape(b, c, h, w)                # groupnorm.py:67-69
        if m.affine:
            y = y * m.weight.view(1, -1, 1, 1) + m.bias.view(1, -1, 1, 1)           # groupnorm.py:70-72
        self.counter += 1
        return y


# ----------------------------------------------------------------------------------------------- Conv2d
class OracleConv2d(_Wrapped):
    def __init__(self, module, cfg, is_first_layer=False):
        super().__init__(module, cfg)
        self.is_first_layer = is_first_layer

    def _first(self, x):                                                            # conv2d.py:20-41
        m, cfg = self.module, self.cfg
        s, p = m.stride[0], m.padding[0]
        H = x.shape[2]
        r = cfg.split_idx()
        units = self.units or [1] * cfg.n_device_per_batch
        rows = self.rows(H // s * units[r] // sum(units))                           # output rows of every rank
        lo, hi = sum(rows[:r]) * s - p, sum(rows[:r + 1]) * s + p
        pad_top, pad_bot = max(0, -lo), max(0, hi - H)
        xs = F.pad(x[:, :, max(lo, 0):min(hi, H)], [p, p, pad_top, pad_bot])
        return F.conv2d(xs, m.weight, m.bias, stride=s)

    def forward(self, x, *args, **kwargs):
        m, cfg = self.module, self.cfg
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        if n == 1:
            y = m(x)                                                                # conv2d.py:51-52
        elif self.is_first_layer:
            y = self._first(x)                                                      # conv2d.py:54-56
        else:
            p = m.padding[0]
            if self.comm is not None and self.idx is None and self.comm.slots is None:
                self.idx = self.comm.register((2, x.shape[0], x.shape[1], p, x.shape[3]))   # conv2d.py:58-65
            if not self._bound():
                y = m(x)                                                            # conv2d.py:68-69
            else:
                edge = torch.stack([x[:, :, :p], x[:, :, -p:]], 0)                  # conv2d.py:90
                sync = cfg.mode == "full_sync" or self._is_sync()
                slots = self.comm.gather_now(self.idx, edge) if sync else self.comm.slots[self.idx]
                zeros = torch.zeros_like(edge[0])
                top = slots[r - 1][1] if r > 0 else zeros                           # conv2d.py:72-88
                bot = slots[r + 1][0] if r < n - 1 else zeros
                y = F.conv2d(torch.cat([top, x, bot], 2), m.weight, m.bias, stride=m.stride[0],
                             padding=(0, m.padding[1]))                             # conv2d.py:95-110
                if not sync and cfg.mode != "no_sync":
                    self.comm.publish(self.idx, edge)                               # conv2d.py:111-112
        self.counter += 1
        return y


# ----------------------------------------------------------------------------------------------- attention
def _heads(t, b, heads):
    return t.view(b, -1, heads, t.shape[-1] // heads).transpose(1, 2)


def _sdpa_out(attn, q, k, v, residual):
    b = q.shape[0]
    o = F.scaled_dot_product_attention(_heads(q, b, attn.heads), _heads(k, b, attn.heads),
                                       _heads(v, b, attn.heads), dropout_p=0.0, is_causal=False)
    o = o.transpose(1, 2).reshape(b, -1, q.shape[-1]).to(q.dtype)
    o = attn.to_out[1](attn.to_out[0](o))                                           # attn.py:93-96,158-161
    if attn.residual_connection:
        o = o + residual
    return o / attn.rescale_output_factor


class OracleSelfAttention(_Wrapped):
    def forward(self, hidden_states, encoder_hidden_states=None, scale=1.0, *args, **kwargs):
        attn, cfg = self.module, self.cfg
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        b, l, _ = hidden_states.shape
        q = attn.to_q(hidden_states)                                                # attn.py:121
        kv = torch.cat([attn.to_k(hidden_states), attn.to_v(hidden_states)], -1)    # attn.py:23-39,125 (fused to_kv)
        if n > 1 and self.comm is not None and self.idx is None and self.comm.slots is None:
            self.idx = self.comm.register((b, l, kv.shape[-1]), self.rows(l))       # attn.py:185-190
        if n == 1:
            full = kv                                                               # attn.py:127-128
        elif not self._bound():
            full = torch.cat([kv] * n, 1)                                           # attn.py:130-131
        elif cfg.mode == "full_sync" or self._is_sync():
            full = torch.cat(self.comm.gather_now(self.idx, kv), 1)                 # attn.py:132-134
        else:
            parts = list(self.comm.slots[self.idx])
            parts[r] = kv                                                           # attn.py:136-138
            full = torch.cat(parts, 1)
            if cfg.mode != "no_sync":
                self.comm.publish(self.idx, kv)                                     # attn.py:139-140
        k, v = full.chunk(2, -1)                                                    # attn.py:142
        out = _sdpa_out(attn, q, k, v, hidden_states)
        self.counter += 1
        return out


class OracleCrossAttention(_Wrapped):
    def __init__(self, module, cfg):
        super().__init__(module, cfg)
        self.kv_cache = None

    def forward(self, hidden_states, encoder_hidden_states=None, scale=1.0, *args, **kwargs):
        assert encoder_hidden_states is not None                                    # attn.py:55
        attn = self.module
        q = attn.to_q(hidden_states)
        if self.counter == 0 or self.kv_cache is None:                              # attn.py:56,73-77
            self.kv_cache = torch.cat([attn.to_k(encoder_hidden_states), attn.to_v(encoder_hidden_states)], -1)
        k, v = self.kv_cache.chunk(2, -1)
        out = _sdpa_out(attn, q, k, v, hidden_states)
        self.counter += 1
        return out


# ----------------------------------------------------------------------------------------------- UNet wrapper
def wrap_unet(model, cfg):
    """Module surgery of DistriUNetPP.__init__ (distri_sdxl_unet_pp.py:18-40)."""
    from diffusers.models.attention_processor import Attention
    if not (cfg.world_size > 1 and cfg.n_device_per_batch > 1):
        return model
    for _, module in list(model.named_modules()):
        if isinstance(module, _Wrapped):
            continue
        for subname, sub in list(module.named_children()):
            if isinstance(sub, nn.Conv2d):
                k = sub.kernel_size
                if k == (1, 1) or k == 1:
                    continue
                setattr(module, subname, OracleConv2d(sub, cfg, is_first_layer=subname == "conv_in"))
            elif isinstance(sub, Attention):
                setattr(module, subname,
                        OracleSelfAttention(sub, cfg) if subname == "attn1" else OracleCrossAttention(sub, cfg))
            elif isinstance(sub, nn.GroupNorm):
                setattr(module, subname, OracleGroupNorm(sub, cfg))
    return model


class OracleUNetPP(nn.Module):
    """Eager path of DistriUNetPP.forward (distri_sdxl_unet_pp.py:117-210) + BaseModel (base_model.py:8-52), with the row
    plan of uneven strips (DistriUNetPP.row_plan)."""

    def __init__(self, model, cfg, bessel=True):
        super().__init__()
        self.model = wrap_unet(model, cfg)
        self.cfg = cfg
        self.comm = None
        self.counter = 0
        self.units = None
        n = cfg.n_device_per_batch
        if cfg.world_size > 1 and n > 1:
            u = 2 ** sum(1 for blk in self.model.down_blocks if getattr(blk, "downsamplers", None) is not None)
            S = cfg.height // 8
            assert S % u == 0 and S // u >= n
            U = S // u
            self.units = [U // n + (1 if k < U % n else 0) for k in range(n)]
        for m in self.wrapped():
            m.units, m.bessel = self.units, bessel

    def wrapped(self):
        return [m for m in self.model.modules() if isinstance(m, _Wrapped)]

    def set_counter(self, c=0):                                                     # base_model.py:27-31
        self.counter = c
        for m in self.wrapped():
            m.set_counter(c)

    def prepare(self, inputs):
        """Buffer sizing + pre-run of the pipeline wrappers (pipelines.py:131-145)."""
        cfg = self.cfg
        if cfg.n_device_per_batch > 1:
            self.comm = OracleComm(cfg)
            for m in self.wrapped():
                m.set_comm(self.comm)
            self.set_counter(0)
            self.forward(**inputs)                       # pass 1: registration
            self.comm.create(inputs["sample"].dtype)
        self.set_counter(0)
        self.forward(**inputs)                           # pass 2: pre-run
        if self.comm is not None:
            self.comm.pending = {}

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None):
        cfg = self.cfg
        B, c, h, w = sample.shape
        if self.comm is not None and self.comm.slots is not None:
            self.comm.begin_step()
        if cfg.world_size == 1:
            out = self.model(sample, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs,
                             return_dict=False)[0]                                  # :118-133
        else:
            split = cfg.do_classifier_free_guidance and cfg.split_batch
            if split:                                                               # :134-146
                assert B == 2
                i = cfg.batch_idx()
                sample = sample[i:i + 1]
                if torch.is_tensor(timestep) and timestep.ndim > 0:
                    timestep = timestep[i:i + 1]
                encoder_hidden_states = encoder_hidden_states[i:i + 1]
                if added_cond_kwargs is not None:
                    added_cond_kwargs = {k: v[i:i + 1] for k, v in added_cond_kwargs.items()}
            out = self.model(sample, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs,
                             return_dict=False)[0].contiguous()
            n = cfg.n_device_per_batch
            if self.units is None or len(set(self.units)) == 1:
                parts = [torch.empty_like(out) for _ in range(cfg.world_size)]
                dist.all_gather(parts, out)                                         # :166,191 (world group)
            else:                                                                   # strips of unequal height
                heights = [h * self.units[q % n] // sum(self.units) for q in range(cfg.world_size)]
                parts = _all_gather_padded(out, heights, 2, None)
            if split:                                                               # :167-168
                out = torch.cat([torch.cat(parts[:n], 2), torch.cat(parts[n:], 2)], 0)
            else:                                                                   # :192
                out = torch.cat(parts, 2)
        self.counter += 1
        return out
