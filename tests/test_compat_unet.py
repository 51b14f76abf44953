"""CPU check that the product's diffusers-compatible UNet (distrifuser_b200/compat) is the same function as the
oracle's diffusers-0.24.0 restatement: identical state-dict keys / shapes / parameter counts and identical fp32
outputs (attention is patched with plain SDPA here -- on the GPU it is always the wgmma kernel)."""
import pytest
import torch
from torch.nn import functional as F

from oracle import workloads


def _sdpa_forward(self, hidden_states, encoder_hidden_states=None, **kw):
    b = hidden_states.shape[0]
    ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
    d = self.inner_dim // self.heads
    q = self.to_q(hidden_states).view(b, -1, self.heads, d).transpose(1, 2)
    k = self.to_k(ctx).view(b, -1, self.heads, d).transpose(1, 2)
    v = self.to_v(ctx).view(b, -1, self.heads, d).transpose(1, 2)
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(b, -1, self.inner_dim)
    return self.to_out[0](o)


@pytest.mark.parametrize("family", ["tiny_sdxl", "tiny_sd15"])
def test_compat_unet_equals_oracle_stub(family, monkeypatch):
    from distrifuser_b200.compat import unet_2d_condition as compat
    monkeypatch.setattr(compat.Attention, "forward", _sdpa_forward)
    ucfg = workloads.unet_config(family)
    ref = workloads.make_unet(family, 0)
    mine = compat.UNet2DConditionModel(**ucfg).eval()
    assert [(k, tuple(v.shape)) for k, v in mine.state_dict().items()] == [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    mine.load_state_dict(ref.state_dict(), strict=True)
    case = workloads.UNetCase("x", family=family)
    inp = workloads.unet_inputs(case, 0, ucfg)
    with torch.no_grad():
        a = ref(**inp, return_dict=False)[0]
        b = mine(inp["sample"].contiguous(memory_format=torch.channels_last), inp["timestep"], inp["encoder_hidden_states"],
                 added_cond_kwargs=inp["added_cond_kwargs"], return_dict=False)[0]
    assert (a - b).abs().max().item() < 2e-5


def test_full_size_parameter_counts():
    """2.567 B (SDXL) and 0.860 B (SD1.x) parameters: the only pin available for the diffusers topology (SURVEY 8c)."""
    from distrifuser_b200.compat import unet_2d_condition as compat
    with torch.device("meta"):
        assert sum(p.numel() for p in compat.UNet2DConditionModel(**compat.SDXL).parameters()) == 2_567_463_684
        assert sum(p.numel() for p in compat.UNet2DConditionModel(**compat.SD15).parameters()) == 859_520_964
        from diffusers.models.unet_2d_condition import UNet2DConditionModel, sd15_config, sdxl_config
        assert sum(p.numel() for p in UNet2DConditionModel(**sdxl_config()).parameters()) == 2_567_463_684
        assert sum(p.numel() for p in UNet2DConditionModel(**sd15_config()).parameters()) == 859_520_964
