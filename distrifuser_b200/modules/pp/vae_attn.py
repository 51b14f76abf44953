"""DistriVAEAttentionPP -- the VAE decoder's mid-block attention (diffusers Attention, one head of width 512) on a row strip.

The inner GroupNorm takes the statistics of the whole image (DistriGroupNorm, exchanged between the ranks), one GEMM computes
q|k|v, the k|v columns are published to every rank synchronously, and df_attn_wide_fwd attends this strip's queries to the
K/V of every strip (its own projection plus the peers' arena slots, read in place); then to_out and the residual."""
import torch
from torch import nn
from torch.nn import functional as F

from ... import _lib
from ...utils import DistriConfig
from ..base_module import BaseModule, nvtx_range
from .groupnorm import DistriGroupNorm


class DistriVAEAttentionPP(BaseModule):
    def __init__(self, module: nn.Module, distri_config: DistriConfig):
        super().__init__(module, distri_config)
        if not (module.heads == 1 and module.to_q.in_features == 512 and module.to_q.out_features == 512):
            raise ValueError(f"the patch-parallel VAE decode runs the decoder's mid-block attention as one head of width 512 "
                             f"(every SD / SDXL VAE); this one has {module.heads} head(s), to_q {module.to_q.in_features} -> "
                             f"{module.to_q.out_features}")
        self.group_norm = DistriGroupNorm(module.group_norm, distri_config)
        self.group_norm.biased_var = True
        self._kvmaps = None
        self._w = None
        self._w_key = None

    def _qkv(self):
        """[to_q ; to_k ; to_v] weights and biases as one [3C, C] GEMM (rebuilt when a source tensor changes)."""
        m = self.module
        src = (m.to_q.weight, m.to_k.weight, m.to_v.weight, m.to_q.bias, m.to_k.bias, m.to_v.bias)
        key = tuple((t._version, t.data_ptr()) for t in src)
        if key != self._w_key:
            with torch.no_grad():
                self._w = (torch.cat(src[:3], 0).contiguous(), torch.cat(src[3:], 0).contiguous())
            self._w_key = key
        return self._w

    @nvtx_range("DistriVAEAttentionPP")
    def forward(self, x: torch.Tensor, temb=None) -> torch.Tensor:
        cfg = self.distri_config
        self._require_cuda_half(x, "DistriVAEAttentionPP")
        m = self.module
        b, c, h, w = x.shape
        n, r = cfg.n_device_per_batch, cfg.split_idx()
        cm = self.comm_manager
        lens = [rows * w for rows in self.patch_rows(h)] if n > 1 else [h * w]
        if n > 1 and self._recording() and self.idx is None:
            self.idx = cm.register_tensor((b, h * w, 2 * c), x.dtype, layer_type="attn",
                                          slot_bytes=b * max(lens) * 2 * c * x.element_size())
        x = x.contiguous(memory_format=torch.channels_last)
        tokens = self.group_norm(x).permute(0, 2, 3, 1).reshape(b, h * w, c)      # NHWC: a view
        wqkv, bqkv = self._qkv()
        qkv = F.linear(tokens, wqkv, bqkv)
        q, kv = qkv[..., :c], qkv[..., c:]
        out = torch.empty((b, h * w, c), dtype=x.dtype, device=x.device)
        L = _lib.lib()
        st = torch.cuda.current_stream().cuda_stream
        live = n > 1 and self._bound()
        if live:
            if self._kvmaps is None:
                self._kvmaps = torch.empty(_lib.NBANKS * n * _lib.TENSORMAP_BYTES, dtype=torch.uint8, device=x.device)
                _lib.check(L.df_attn_wide_make_kvmaps(cm.group, cm.tensor_off[self.idx], cm.slot_bytes[self.idx], b,
                                                      _lib.int32_array(lens), c, self._kvmaps.data_ptr(), st),
                           "df_attn_wide_make_kvmaps")
            cm.enqueue(self.idx, kv, async_stream=False)
            comm, maps, nseg, own, idx = cm.group, self._kvmaps.data_ptr(), n, r, self.idx
        else:
            # one rank, or the registration pass before the buffers exist (its value is never used)
            comm, maps, nseg, own, idx, lens = _lib.null_comm(), None, 1, 0, 0, [h * w]
        _lib.check(L.df_attn_wide_fwd(comm, q.data_ptr(), kv.data_ptr(), out.data_ptr(), maps, b, h * w, _lib.int32_array(lens),
                                      c, q.stride(1), kv.stride(1), out.stride(1), nseg, own, _lib.int32_array(range(_lib.MAX_WORLD)),
                                      idx, int(live), 0.0, st), "df_attn_wide_fwd")
        o = m.to_out[1](F.linear(out, m.to_out[0].weight, m.to_out[0].bias))
        o = o.reshape(b, h, w, c).permute(0, 3, 1, 2)                             # channels_last NCHW view
        if m.residual_connection:
            o = o + x
        if m.rescale_output_factor != 1.0:
            o = o / m.rescale_output_factor
        self.counter += 1
        return o
