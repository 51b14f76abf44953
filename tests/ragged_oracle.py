"""TEST INFRASTRUCTURE -- the CPU oracle (oracle/pp_modules.py, fp32) extended to uneven row strips.

The reference asserts equal strips, so it cannot pin this: these classes restate the product's uneven rule on top of the
oracle's reference restatement and change nothing for equal strips (every path below falls back to the parent class's,
or to its exact formula).  Patch rank r of n holds `units[r]` units of 2^downsamplers latent rows
(U // n, one more for the first U % n ranks; distrifuser_b200.utils.split_units):

  * K/V segments of unequal length: RaggedComm gathers tensors whose dim 1 differs between ranks;
  * GroupNorm: every mean over ranks weighs rank s by rows_s / sum(rows) (sync, corrected_async_gn, stale_gn, and the
    all-reduce of sync_gn / full_sync);
  * conv_in slice and final gather at the prefix sums of the rows.

`bessel=False` drops the local-count Bessel factor, so that an uneven full_sync run equals the one-device UNet exactly."""
from __future__ import annotations

import torch
from torch import distributed as dist
from torch import nn
from torch.nn import functional as F

from oracle.pp_modules import (OracleComm, OracleConv2d, OracleCrossAttention, OracleGroupNorm, OracleSelfAttention,
                               OracleUNetPP, _moments, _Wrapped)


def all_gather_var(local: torch.Tensor, n: int, dim: int, group) -> list[torch.Tensor] | None:
    """The n members' tensors when they differ in size along `dim` (uneven strips), else None (use a plain all_gather)."""
    size = torch.tensor([local.shape[dim]])
    sizes = [torch.zeros_like(size) for _ in range(n)]
    dist.all_gather(sizes, size, group=group)
    sizes = [int(t) for t in sizes]
    if len(set(sizes)) == 1:
        return None
    shape = list(local.shape)
    shape[dim] = max(sizes)
    padded = local.new_zeros(shape)
    padded.narrow(dim, 0, local.shape[dim]).copy_(local)
    bufs = [torch.empty_like(padded) for _ in range(n)]
    dist.all_gather(bufs, padded, group=group)
    return [b.narrow(dim, 0, sz).contiguous() for b, sz in zip(bufs, sizes)]


class RaggedComm(OracleComm):
    """OracleComm whose slots may hold tensors of different lengths per source (K/V of uneven strips)."""

    def _gather_into(self, idx: int, local: torch.Tensor):
        parts = all_gather_var(local, self.n, 1, self.cfg.batch_group)
        if parts is None:
            dist.all_gather(self.slots[idx], local, group=self.cfg.batch_group)
        else:
            self.slots[idx] = parts

    def gather_now(self, idx: int, local: torch.Tensor):
        self._gather_into(idx, local.contiguous())
        return self.slots[idx]

    def begin_step(self):
        for idx in sorted(self.pending):
            self._gather_into(idx, self.pending[idx])
        self.pending = {}


class _Rows:
    """Row plan of a wrapper: set by RaggedUNetPP (None: equal strips)."""
    units: list[int] | None = None
    bessel: bool = True

    def rows(self, h):
        """Rows of every patch rank where this rank holds h rows (tokens alike): distrifuser_b200.utils.patch_rows."""
        n, r = self.cfg.n_device_per_batch, self.cfg.split_idx()
        units = self.units or [1] * n
        return [u * h // units[r] for u in units]

    def uneven(self):
        return self.units is not None and len(set(self.units)) > 1


class RaggedGroupNorm(_Rows, OracleGroupNorm):
    def forward(self, x):
        if not self.uneven() and self.bessel:
            return super().forward(x)
        m, cfg = self.module, self.cfg
        b, c, h, w = x.shape
        G = m.num_groups
        stat_modes = cfg.mode in ("stale_gn", "corrected_async_gn")
        if stat_modes and self.comm is not None and self.idx is None and self.comm.slots is None:
            self.idx = self.comm.register((2, b, G, 1, 1, 1))
        if not stat_modes and not (self._is_sync() or cfg.mode in ("sync_gn", "full_sync")):
            self.counter += 1
            return m(x)
        x5 = x.reshape(b, G, c // G, h, w)
        mine = _moments(x5)
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        rows = self.rows(h)
        wts = [s / sum(rows) for s in rows]                                         # each rank's share of the rows
        use_local_fallback = False
        if stat_modes:
            if not self._bound():
                full = mine
            elif self._is_sync():
                full = sum(wt * g for wt, g in zip(wts, self.comm.gather_now(self.idx, mine)))
            else:
                stale = self.comm.slots[self.idx]
                if cfg.mode == "corrected_async_gn":
                    full = sum(wt * g for wt, g in zip(wts, stale)) + (mine - stale[r])
                else:
                    full = sum(wt * (mine if s == r else g) for s, (wt, g) in enumerate(zip(wts, stale)))
                self.comm.publish(self.idx, mine)
            if cfg.mode == "corrected_async_gn":
                use_local_fallback = True
        else:
            full = mine * wts[r]
            if n > 1:
                dist.all_reduce(full, op=dist.ReduceOp.SUM, group=cfg.batch_group)
        mean, meansq = full[0], full[1]
        var = meansq - mean * mean
        if use_local_fallback:
            var = torch.where(var < 0, mine[1] - mine[0] * mine[0], var)
        ne = (c // G) * h * w
        if self.bessel:
            var = var * (ne / (ne - 1))
        y = ((x5 - mean) / (var + m.eps).sqrt()).reshape(b, c, h, w)
        if m.affine:
            y = y * m.weight.view(1, -1, 1, 1) + m.bias.view(1, -1, 1, 1)
        self.counter += 1
        return y


class RaggedConv2d(_Rows, OracleConv2d):
    def _first(self, x):
        """conv_in slice of this rank's rows, starting at the prefix sum of the lower ranks' rows."""
        m, cfg = self.module, self.cfg
        s, p = m.stride[0], m.padding[0]
        H = x.shape[2]
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        units = self.units or [1] * n
        rows = self.rows(H // s * units[r] // sum(units))
        lo, hi = sum(rows[:r]) * s - p, sum(rows[:r + 1]) * s + p
        pad_top, pad_bot = max(0, -lo), max(0, hi - H)
        xs = F.pad(x[:, :, max(lo, 0):min(hi, H)], [p, p, pad_top, pad_bot])
        return F.conv2d(xs, m.weight, m.bias, stride=s)


def wrap_unet(model, cfg):
    """oracle.pp_modules.wrap_unet with the ragged GroupNorm / conv wrappers (attention needs only RaggedComm)."""
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
                setattr(module, subname, RaggedConv2d(sub, cfg, is_first_layer=subname == "conv_in"))
            elif isinstance(sub, Attention):
                setattr(module, subname,
                        OracleSelfAttention(sub, cfg) if subname == "attn1" else OracleCrossAttention(sub, cfg))
            elif isinstance(sub, nn.GroupNorm):
                setattr(module, subname, RaggedGroupNorm(sub, cfg))
    return model


class RaggedUNetPP(OracleUNetPP):
    """OracleUNetPP with the product's row plan (DistriUNetPP.row_plan) and a gather of unequal strips."""

    def __init__(self, model, cfg, bessel=True):
        nn.Module.__init__(self)
        self.model = wrap_unet(model, cfg)
        self.cfg = cfg
        self.comm = None
        self.counter = 0
        n = cfg.n_device_per_batch
        self.units = None
        if cfg.world_size > 1 and n > 1:
            u = 2 ** sum(1 for blk in self.model.down_blocks if getattr(blk, "downsamplers", None) is not None)
            S = cfg.height // 8
            assert S % u == 0 and S // u >= n
            U = S // u
            self.units = [U // n + (1 if k < U % n else 0) for k in range(n)]
        for m in self.wrapped():
            m.units, m.bessel = self.units, bessel

    def prepare(self, inputs):
        cfg = self.cfg
        if cfg.n_device_per_batch > 1:
            self.comm = RaggedComm(cfg)
            for m in self.wrapped():
                m.set_comm(self.comm)
            self.set_counter(0)
            self.forward(**inputs)
            self.comm.create(inputs["sample"].dtype)
        self.set_counter(0)
        self.forward(**inputs)
        if self.comm is not None:
            self.comm.pending = {}

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None):
        cfg = self.cfg
        B = sample.shape[0]
        if self.comm is not None and self.comm.slots is not None:
            self.comm.begin_step()
        if cfg.world_size == 1:
            out = self.model(sample, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs, return_dict=False)[0]
        else:
            split = cfg.do_classifier_free_guidance and cfg.split_batch
            if split:
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
            parts = all_gather_var(out, cfg.world_size, 2, None)                    # strips of unequal height
            if parts is None:
                parts = [torch.empty_like(out) for _ in range(cfg.world_size)]
                dist.all_gather(parts, out)
            n = cfg.n_device_per_batch
            if split:
                out = torch.cat([torch.cat(parts[:n], 2), torch.cat(parts[n:], 2)], 0)
            else:
                out = torch.cat(parts, 2)
        self.counter += 1
        return out
