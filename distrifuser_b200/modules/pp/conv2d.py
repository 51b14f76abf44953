"""DistriConv2dPP -- drop-in for distrifuser/modules/pp/conv2d.py:10-115.

The halo rows go to the two patch neighbours only (df_halo_push, peer stores over NVLink) instead of an
all_gather over every rank, and the padded conv input is assembled by one vectorised kernel
(df_halo_assemble) instead of torch.stack + cat + F.pad.  The convolution itself stays a cuDNN library call
on the NHWC padded tensor (SURVEY 8f N1 lists the hand-written implicit GEMM as a later row)."""
import torch
from torch import nn
from torch.nn import functional as F

from ... import _lib, ops
from ...utils import DistriConfig, patch_rows, row_offset
from ..base_module import BaseModule, nvtx_range


class DistriConv2dPP(BaseModule):
    def __init__(self, module: nn.Conv2d, distri_config: DistriConfig, is_first_layer: bool = False):
        super().__init__(module, distri_config)
        self.is_first_layer = is_first_layer

    def _conv(self, x: torch.Tensor, padding, residual=None, fold_bias=False, bias=None) -> torch.Tensor:
        """F.conv2d(x, weight, bias, stride, padding) (+ residual): cuDNN without bias + one vectorised bias / residual pass."""
        return ops.conv2d_bias_residual(x, self.module, padding, residual=residual, bias=bias, fold_bias=fold_bias)

    def naive_forward(self, x: torch.Tensor, residual=None, fold_bias=False, bias=None) -> torch.Tensor:        # conv2d.py:15-18
        return self._conv(x, self.module.padding, residual, fold_bias, bias)

    def sliced_forward(self, x: torch.Tensor) -> torch.Tensor:       # conv2d.py:20-41 (conv_in: 4 channels, tiny)
        cfg = self.distri_config
        b, c, h, w = x.shape
        n = cfg.n_device_per_batch
        units = self.row_units or [1] * n
        stride, padding = self.module.stride[0], self.module.padding[0]
        assert h // stride % sum(units) == 0
        r = cfg.split_idx()
        rows = patch_rows(units, r, h // stride * units[r] // sum(units))      # every rank's output rows (prefix sums: uneven strips)
        lo, hi = row_offset(rows, r) * stride - padding, row_offset(rows, r + 1) * stride + padding
        pad_t, pad_b = max(0, -lo), max(0, hi - h)
        xs = F.pad(x[:, :, max(lo, 0):min(hi, h), :], [padding, padding, pad_t, pad_b])
        return F.conv2d(xs, self.module.weight, self.module.bias, stride=stride, padding="valid")     # 4 input channels: tiny

    # -- GroupNorm-fused halo path (the producer's normalise pass writes the padded conv input, ships the boundary rows and fills
    #    the margins: no df_halo_push / df_halo_assemble launches and no copy of the whole activation)
    def halo_plan(self, x: torch.Tensor):
        """-> (idx, tensor_off, slot_bytes, up, down, push) when this conv can take a padded input produced by its GroupNorm in
        the current call, else None (one patch, first layer, buffers not created yet, not 3x3 / padding 1)."""
        cfg = self.distri_config
        n = cfg.n_device_per_batch
        if n == 1 or self.is_first_layer or not self._bound():
            return None
        m = self.module
        if m.padding[0] != 1 or m.kernel_size[0] != 3 or m.padding[1] != 1:
            return None
        cm = self.comm_manager
        r = cfg.split_idx()
        up, down = (r - 1 if r > 0 else -1), (r + 1 if r < n - 1 else -1)
        sync = cfg.mode == "full_sync" or self._is_sync_step()
        push = sync or cfg.mode != "no_sync"                         # conv2d.py:92-93 / :111-112
        return self.idx, cm.tensor_off[self.idx], cm.slot_bytes[self.idx], up, down, push

    @nvtx_range("DistriConv2dPP")
    def forward_padded(self, xp: torch.Tensor, residual=None, fold_bias=False, bias=None) -> torch.Tensor:
        """xp: [b, C, h+2, w] NHWC with the halo rows in place (DistriGroupNorm.forward(..., pad_for=self))."""
        out = self._conv(xp, (0, self.module.padding[1]), residual, fold_bias, bias)   # conv2d.py:95-110
        self.counter += 1
        return out

    @nvtx_range("DistriConv2dPP")
    def forward(self, x: torch.Tensor, *args, residual=None, fold_bias=False, bias=None, **kwargs) -> torch.Tensor:
        """residual / bias / fold_bias (extensions, see ops.conv2d_bias_residual): `conv(x) + bias + residual` in one pass after
        the convolution (bias: a vector replacing module.bias); fold_bias = the caller accounts for the bias elsewhere."""
        cfg = self.distri_config
        n = cfg.n_device_per_batch
        if n == 1:
            out = self.naive_forward(x, residual, fold_bias, bias)   # conv2d.py:51-52
        elif self.is_first_layer:
            assert residual is None and not fold_bias
            out = self.sliced_forward(x)                             # conv2d.py:54-56
        else:
            self._require_cuda_half(x, "DistriConv2dPP")
            p = self.module.padding[0]
            b, c, h, w = x.shape
            if self._recording() and self.idx is None:
                self.idx = self.comm_manager.register_tensor([2, b, c, p, w], x.dtype, layer_type="conv2d")  # :58-65
            if not self._bound():
                out = self.naive_forward(x, residual, fold_bias, bias)   # conv2d.py:68-69
            else:
                assert p == 1 and self.module.kernel_size[0] == 3, "halo exchange is written for 3x3 / padding 1"
                cm = self.comm_manager
                L = _lib.lib()
                r = cfg.split_idx()
                up, down = (r - 1 if r > 0 else -1), (r + 1 if r < n - 1 else -1)
                x = x.contiguous(memory_format=torch.channels_last)
                xp = torch.empty((b, c, h + 2, w), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
                st = torch.cuda.current_stream().cuda_stream
                off, sb = cm.tensor_off[self.idx], cm.slot_bytes[self.idx]
                sync = cfg.mode == "full_sync" or self._is_sync_step()
                dt = _lib.dtype_code(x.dtype)                        # fp16, or fp32 in the VAE decoder's upcast part
                if sync:                                             # conv2d.py:92-93: fresh halos
                    _lib.check(L.df_halo_push_dtype(cm.group, x.data_ptr(), b, h, w, c, self.idx, off, sb, up, down, dt, st),
                               "df_halo_push_dtype")
                _lib.check(L.df_halo_assemble_dtype(cm.group, x.data_ptr(), xp.data_ptr(), b, h, w, c, self.idx, off, sb,
                                                    up, down, 1, dt, st), "df_halo_assemble_dtype")
                out = self._conv(xp, (0, self.module.padding[1]), residual, fold_bias, bias)   # conv2d.py:95-110
                if not sync and cfg.mode != "no_sync":               # conv2d.py:111-112: ship for the next step
                    _lib.check(L.df_halo_push_dtype(cm.group, x.data_ptr(), b, h, w, c, self.idx, off, sb, up, down, dt, st),
                               "df_halo_push_dtype")
        self.counter += 1
        return out
