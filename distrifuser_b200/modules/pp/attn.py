"""DistriSelfAttentionPP / DistriCrossAttentionPP -- drop-ins for distrifuser/modules/pp/attn.py:12-195.

q / fused q|k|v / out projections are cuBLAS GEMMs unless DF_LINEAR puts them on the hand-written one (ops.linear /
ops.project); everything between them --
the reference's torch.cat of the per-rank K/V (attn.py:131-138), split / view / transpose (:142-149) and
F.scaled_dot_product_attention (:153) -- is one wgmma kernel (df_attn_fwd) that TMA-loads the K/V tiles
straight from the n per-rank segments: this rank's fresh projection and the peers' 1-step-stale arena slots."""
import ctypes as C

import torch
from torch import nn
from torch.nn import functional as F

from ... import _lib
from ...utils import DistriConfig
from ..base_module import BaseModule, nvtx_range


_WORKSPACES: dict = {}      # device -> list of zero-initialised scratch tensors (kept alive: captured graphs hold raw pointers)


def _shared_workspace(device, nbytes: int) -> torch.Tensor:
    """Scratch of the attention schedule (work-unit ticket counter, fp32 partials + arrival tickets of split units: df_attn_workspace_bytes).
    One buffer per device serves every attention layer: the launches are ordered on one stream.  It must start zeroed."""
    lst = _WORKSPACES.setdefault(device, [])
    if not lst or lst[-1].numel() < nbytes:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("attention workspace would grow during CUDA-graph capture; run one eager UNet call first")
        lst.append(torch.zeros(max(nbytes, 16 << 20), dtype=torch.uint8, device=device))
    return lst[-1]


class DistriAttentionPP(BaseModule):
    def __init__(self, module: nn.Module, distri_config: DistriConfig):
        super().__init__(module, distri_config)
        to_k, to_v = module.to_k, module.to_v                            # attn.py:16-21
        assert isinstance(to_k, nn.Linear) and isinstance(to_v, nn.Linear)
        assert (to_k.bias is None) == (to_v.bias is None)
        assert to_k.weight.shape == to_v.weight.shape
        in_size, out_size = to_k.in_features, to_k.out_features
        to_kv = nn.Linear(in_size, out_size * 2, bias=to_k.bias is not None, device=to_k.weight.device,
                          dtype=to_k.weight.dtype)                       # attn.py:23-39 (K | V fused)
        with torch.no_grad():
            to_kv.weight[:out_size].copy_(to_k.weight)
            to_kv.weight[out_size:].copy_(to_v.weight)
            if to_k.bias is not None:
                to_kv.bias[:out_size].copy_(to_k.bias)
                to_kv.bias[out_size:].copy_(to_v.bias)
        self.to_kv = to_kv
        self._kvmaps = None

    def _attend(self, q, kv_own, lens, own_seg, wait_flags, kind="self", scale=0.0, real_width=None):
        """softmax(q k^T * scale) v over the K/V segments of `lens[s]` rows (the patch ranks' strips, unequal when the strips
        are); q:[b,lq,C], kv_own:[b,lens[own_seg],2C]; scale 0 = 1/sqrt(d) of the stored head width (pass it explicitly when the
        heads are zero-padded)."""
        attn = self.module
        b, lq, Cq = q.shape
        heads = attn.heads
        d = Cq // heads
        out = torch.empty((b, lq, Cq), dtype=q.dtype, device=q.device)
        cm = self.comm_manager
        nseg = len(lens)
        if nseg > 1:
            comm, maps = cm.group, self._kvmaps.data_ptr()
        else:
            comm, maps = _lib.null_comm(), None
        seg_rank = (C.c_int32 * _lib.MAX_WORLD)(*range(_lib.MAX_WORLD))
        seg_len = _lib.int32_array(lens)
        L = _lib.lib()
        ws_bytes = L.df_attn_workspace_bytes_ragged(b, lq, seg_len, nseg, heads, d)
        ws = _shared_workspace(q.device, ws_bytes).data_ptr() if ws_bytes else None
        prof = _lib.PROFILE
        if prof is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        _lib.check(L.df_attn_fwd_ragged(comm, q.data_ptr(), kv_own.data_ptr(), out.data_ptr(), maps, b, lq, seg_len,
                                        heads, d, q.stride(1), kv_own.stride(1), out.stride(1), nseg, own_seg,
                                        seg_rank, self.idx or 0, int(wait_flags), float(scale), ws, ws_bytes,
                                        torch.cuda.current_stream().cuda_stream), "df_attn_fwd_ragged")
        if prof is not None:
            e1.record()
            prof.append(dict(kernel="fmha_fwd_kernel", kind=kind,
                             flops=4.0 * b * lq * sum(lens) * (real_width or Cq),   # algorithmic: zero-padded head columns do not count
                             bytes=2.0 * (2 * b * lq * Cq + b * sum(lens) * 2 * Cq),
                             shape=(b, lq, sum(lens), heads, d), start=e0, end=e1))
        return out

    def _project_out(self, hidden_states, residual, weight=None):
        from ... import ops
        attn = self.module
        # attn.py:93-96 / 158-161; weight: to_out with zero columns for the padded head dims (see _qkv_weight)
        hidden_states = ops.project("out", hidden_states, attn.to_out[0], weight)
        hidden_states = attn.to_out[1](hidden_states)
        if attn.residual_connection:
            hidden_states = hidden_states + residual
        if attn.rescale_output_factor != 1.0:
            hidden_states = hidden_states / attn.rescale_output_factor
        return hidden_states


class DistriCrossAttentionPP(DistriAttentionPP):
    def __init__(self, module: nn.Module, distri_config: DistriConfig):
        super().__init__(module, distri_config)
        self.kv_cache = None

    @nvtx_range("DistriCrossAttentionPP")
    def forward(self, hidden_states, encoder_hidden_states=None, scale: float = 1.0, *args, **kwargs):
        assert encoder_hidden_states is not None                         # attn.py:55
        self._require_cuda_half(hidden_states, "DistriCrossAttentionPP")
        attn = self.module
        from ... import ops
        q = ops.project("qkv", hidden_states, attn.to_q)
        if self.counter == 0 or self.kv_cache is None:                   # attn.py:56,73-77: text K/V once per image
            kv = self.to_kv(encoder_hidden_states)
            if self.kv_cache is not None and self.kv_cache.shape == kv.shape:
                self.kv_cache.copy_(kv)                                  # stable address for captured graphs
            else:
                self.kv_cache = kv
        kv = self.kv_cache
        out = self._attend(q, kv, [kv.shape[1]], 0, False, kind="cross")
        out = self._project_out(out, hidden_states)
        self.counter += 1
        return out


class DistriSelfAttentionPP(DistriAttentionPP):
    def __init__(self, module: nn.Module, distri_config: DistriConfig):
        super().__init__(module, distri_config)
        # q and k|v read the same activations: one [C -> 3C] GEMM instead of two launches (to_kv is kept: it is the reference's
        # attribute, attn.py:39, and sizes the registered slot)
        self._w_qkv = None
        self._w_qkv_key = None
        self._w_out = None               # to_out weight with zero columns for the padded head dims (d < 64 only)
        self._head_pad = 0               # stored head width when the heads are padded (64), else 0

    def _qkv_weight(self, dtype):
        """[to_q.weight ; to_kv.weight] as one [3C, C] matrix, rebuilt whenever either source changed (load_state_dict,
        LoRA fuse/unfuse, in-place edits, .to()/.half()): the key holds the tensors' version counters and storage.
        Heads narrower than 64 (SD1.x level 0: d = 40) are stored 64 wide -- zero rows in the projection, zero columns in
        to_out, the softmax scale passed explicitly: an 80-byte head row at offset 80*h of the token row costs the TMA 1.6 cache
        lines per row request and leaves the kernel waiting for K/V tiles; 128-byte rows are one line each."""
        to_q, to_kv = self.module.to_q, self.to_kv
        if not (isinstance(to_q, nn.Linear) and to_q.bias is None and to_kv.bias is None and
                to_q.in_features == to_kv.in_features and to_q.out_features * 2 == to_kv.out_features and
                to_q.weight.dtype == dtype and to_kv.weight.dtype == dtype):
            return None
        wq, wkv, wo = to_q.weight, to_kv.weight, self.module.to_out[0].weight
        heads = self.module.heads
        d = to_q.out_features // heads
        pad = 64 if d < 64 else 0
        key = (wq._version, wkv._version, wo._version, wq.data_ptr(), wkv.data_ptr(), wo.data_ptr(), wq.device, dtype, pad)
        if key != self._w_qkv_key:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("DistriSelfAttentionPP: attention weights changed since the last eager call; run one "
                                   "eager UNet call (pipeline.prepare()) before capturing CUDA graphs")
            with torch.no_grad():
                if pad:
                    cin = wq.shape[1]
                    widen = lambda w: F.pad(w.detach().reshape(-1, heads, d, cin), (0, 0, 0, pad - d)).reshape(-1, cin)
                    self._w_qkv = torch.cat([widen(wq), widen(wkv)], 0).contiguous()          # [3 * heads * 64, C]
                    self._w_out = F.pad(wo.detach().reshape(wo.shape[0], heads, d), (0, pad - d)).reshape(wo.shape[0], heads * pad).contiguous()
                else:
                    self._w_qkv = torch.cat([wq.detach(), wkv.detach()], 0).contiguous()
                    self._w_out = None
            self._w_qkv_key = key
            self._head_pad = pad
        return self._w_qkv

    @nvtx_range("DistriSelfAttentionPP")
    def forward(self, hidden_states, encoder_hidden_states=None, scale: float = 1.0, *args, **kwargs):
        cfg = self.distri_config
        self._require_cuda_half(hidden_states, "DistriSelfAttentionPP")
        attn = self.module
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        b, l, c = hidden_states.shape
        cm = self.comm_manager
        w_qkv = self._qkv_weight(hidden_states.dtype)
        heads = attn.heads
        d_real = c // heads
        padded = w_qkv is not None and self._head_pad != 0
        cs = heads * self._head_pad if padded else c                     # stored width of q (and of each of k, v)
        lens = self.patch_rows(l) if n > 1 else [l]                      # tokens of every rank's strip (unequal strips differ)
        if n > 1 and self._recording() and self.idx is None:
            # every rank's slot has the size of the LARGEST strip's K/V, so that all ranks compute the same arena layout
            self.idx = cm.register_tensor((b, l, 2 * cs), hidden_states.dtype, layer_type="attn",                 # :185-190
                                          slot_bytes=b * max(lens) * 2 * cs * hidden_states.element_size())
        live = n > 1 and self._bound()
        sync = live and (cfg.mode == "full_sync" or self._is_sync_step())
        ship = live and (sync or cfg.mode != "no_sync")                  # attn.py:133 / :139-140
        published = False
        if w_qkv is not None:
            from ... import ops
            if not padded and ops.use_fused_linear("qkv") and ops.linear_supported(b * l, 3 * c, c):
                # hand-written wgmma GEMM; its epilogue stores the k|v columns straight into the peers' arena slots and the
                # last CTA stamps their flags: no enqueue copy (utils.py:187), no separate publication kernel
                pub = (cm.group, c, self.idx, cm.peers_mask(), cm.tensor_off[self.idx], cm.slot_bytes[self.idx]) if ship else None
                qkv = ops.linear(hidden_states, w_qkv, publish=pub)
                published = ship
            else:
                qkv = F.linear(hidden_states, w_qkv)                     # attn.py:121,125 in one GEMM
            q, kv = qkv[..., :cs], qkv[..., cs:]                         # views: row pitch 3C, no copies
        else:
            q = attn.to_q(hidden_states)                                 # attn.py:121
            kv = self.to_kv(hidden_states)                               # attn.py:125
        sm_scale = d_real ** -0.5 if padded else 0.0
        if not live:
            # attn.py:127-131: one rank, or buffers not created yet (n identical copies of kv give the same softmax)
            out = self._attend(q, kv, [l], 0, False, scale=sm_scale, real_width=c)
        else:
            if self._kvmaps is None:
                self._kvmaps = torch.empty(_lib.NBANKS * n * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device=q.device)
                _lib.check(_lib.lib().df_attn_make_kvmaps_ragged(cm.group, cm.tensor_off[self.idx], cm.slot_bytes[self.idx], b,
                                                                 _lib.int32_array(lens), heads, cs // heads,
                                                                 self._kvmaps.data_ptr(), torch.cuda.current_stream().cuda_stream),
                           "df_attn_make_kvmaps_ragged")
            if ship and not published:
                cm.enqueue(self.idx, kv, async_stream=not sync)          # sync: everyone needs it this step; async: hidden
            out = self._attend(q, kv, lens, r, True, scale=sm_scale, real_width=c)   # attn.py:134-153, peers' segments in place
        out = self._project_out(out, hidden_states, self._w_out if padded else None)
        self.counter += 1
        return out
