"""CPU checks of the diffusers stand-ins used when `diffusers` is absent (distrifuser_b200/compat): scheduler constants of
the SD/SDXL configuration and the denoising-loop plumbing of the latent pipeline (CFG duplication, guidance combine)."""
import math

import torch

from distrifuser_b200.compat.pipeline import SyntheticLatentPipeline
from distrifuser_b200.compat.schedulers import DDIMScheduler, EulerDiscreteScheduler


def test_euler_schedule_constants():
    s = EulerDiscreteScheduler()
    s.set_timesteps(50)
    assert s.timesteps.tolist()[0] == 981 and s.timesteps.tolist()[-1] == 1            # "leading" spacing, steps_offset 1
    sig = s.sigmas
    assert len(sig) == 51 and sig[-1] == 0 and all(sig[i] > sig[i + 1] for i in range(50))
    # sqrt(sigma_max^2 + 1) over the SELECTED timesteps (t=981 -> 13.16; 14.6 is the value before set_timesteps, t=999)
    assert abs(s.init_noise_sigma - math.sqrt(float(sig[0]) ** 2 + 1)) < 1e-5 and 13.0 < s.init_noise_sigma < 13.4
    x = torch.randn(1, 4, 8, 8)
    assert torch.allclose(s.scale_model_input(x), x / math.sqrt(float(sig[0]) ** 2 + 1))
    prev = s.step(torch.ones_like(x), s.timesteps[0], x)[0]
    assert torch.allclose(prev, x + (float(sig[1]) - float(sig[0])))


def test_ddim_step_is_identity_for_consistent_eps():
    s = DDIMScheduler()
    s.set_timesteps(50)
    x0 = torch.randn(1, 4, 8, 8)
    eps = torch.randn(1, 4, 8, 8)
    t = int(s._ts_host[0])
    a = float(s.alphas_cumprod[t])
    xt = a ** 0.5 * x0 + (1 - a) ** 0.5 * eps
    prev = s.step(eps, s.timesteps[0], xt)[0]
    a_prev = float(s.alphas_cumprod[t - s._ratio])
    assert torch.allclose(prev, a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * eps, atol=1e-5)


class _FakeUNet:
    """Returns eps = cond-dependent constant so the CFG combine is observable; records the calls it receives."""

    def __init__(self):
        from types import SimpleNamespace
        self.config = SimpleNamespace(in_channels=4, cross_attention_dim=16, projection_class_embeddings_input_dim=6 * 8 + 12,
                                      addition_time_embed_dim=8)
        self.calls = []

    def __call__(self, x, t, encoder_hidden_states=None, added_cond_kwargs=None, return_dict=False):
        self.calls.append((tuple(x.shape), float(t), tuple(encoder_hidden_states.shape),
                           None if added_cond_kwargs is None else tuple(added_cond_kwargs["time_ids"].shape)))
        eps = torch.zeros_like(x)
        if x.shape[0] == 2:
            eps[1] = 1.0                      # cond branch predicts 1, uncond 0 -> combined = guidance_scale
        return (eps,)


def test_latent_pipeline_loop_and_cfg():
    unet = _FakeUNet()
    pipe = SyntheticLatentPipeline(unet, sdxl=True, device="cpu", dtype=torch.float32)
    g = torch.Generator().manual_seed(0)
    out = pipe(prompt="x", height=64, width=64, num_inference_steps=5, guidance_scale=5.0, generator=g).images
    assert out.shape == (1, 4, 8, 8) and len(unet.calls) == 5
    shp, t0, ehs, ids = unet.calls[0]
    assert shp == (2, 4, 8, 8) and ehs == (2, 77, 16) and ids == (2, 6)                 # CFG batch duplication, SDXL time ids
    assert [c[1] for c in unet.calls] == sorted([c[1] for c in unet.calls], reverse=True)
    # with eps == guidance_scale everywhere, Euler gives x_T + 5 * (0 - sigma_0)
    s = EulerDiscreteScheduler(); s.set_timesteps(5)
    g2 = torch.Generator().manual_seed(0)
    x_T = torch.randn((1, 4, 8, 8), generator=g2) * s.init_noise_sigma
    assert torch.allclose(out, x_T - 5.0 * float(s.sigmas[0]), atol=1e-4)
    # guidance off: single batch, no duplication
    unet.calls.clear()
    pipe(prompt="x", height=64, width=64, num_inference_steps=2, guidance_scale=1.0, generator=g)
    assert unet.calls[0][0] == (1, 4, 8, 8)


def test_launch_summarizer_families(tmp_path):
    import importlib.util, os, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("summ", os.path.join(root, "tools", "summarize_launches.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    assert m.family("void <unnamed>::fmha_fwd_kernel<1>(CUtensorMap_st ...)").startswith("OURS fmha")
    assert m.family("<unnamed>::add_layernorm_kernel<5>(...)").startswith("OURS add_layernorm")
    assert m.family("nvjet_hsh_192x256_64x5_2x1_2cta_v_bz_bias_TNT") == "library GEMM (cuBLAS)"
    assert "elementwise" in m.family("void at::vectorized_elementwise_kernel<8, at::CUDAFunctor_add<c10::Half>>")
    # cuDNN's sm100 convolutions are cutlass3x "... implicit_gemm_fprop ..." kernels: they must not be booked as cuBLAS (round-1 bug)
    assert m.family("cutlass3x_sm100_tensorop_s256x256x16implicit_gemm_fprop_f16_f16_f32_void_f16_...") == "library conv (cuDNN)"
    assert m.family("void <unnamed>::linear_kernel<1, 256>(CUtensorMap_st, CUtensorMap_st, <unnamed>::LinearArgs)").startswith("OURS wgmma GEMM")
    assert m.family("<unnamed>::gn_fused_kernel(const __half *, ...)").startswith("OURS gn_fused")


def test_geglu_interleave_layout():
    """Rows of the fused GEGLU weight: [hidden block t | gate block t] per tile (ops.geglu_interleave), blocks of 80 / 128."""
    import torch
    from distrifuser_b200 import ops
    for block, D in ((128, 512), (80, 320)):
        w = torch.arange(2 * D * 3, dtype=torch.float32).reshape(2 * D, 3)
        b = torch.arange(2 * D, dtype=torch.float32)
        wi, bi = ops.geglu_interleave(w, b, block)
        for t in range(D // block):
            assert torch.equal(wi[2 * t * block:(2 * t + 1) * block], w[t * block:(t + 1) * block])                 # hidden
            assert torch.equal(wi[(2 * t + 1) * block:(2 * t + 2) * block], w[D + t * block:D + (t + 1) * block])   # gate
            assert torch.equal(bi[(2 * t + 1) * block:(2 * t + 2) * block], b[D + t * block:D + (t + 1) * block])


def test_batched_time_embedding_is_noop_on_cpu():
    """compat UNet: the one-GEMM time-embedding projection is a CUDA fp16 fast path; on CPU every block projects itself."""
    import torch
    from distrifuser_b200.compat.unet_2d_condition import SD15, UNet2DConditionModel
    cfg = dict(SD15, block_out_channels=(32, 64), down_block_types=("DownBlock2D", "DownBlock2D"), up_block_types=("UpBlock2D", "UpBlock2D"),
               attention_head_dim=(2, 2), transformer_layers_per_block=(1, 1), norm_num_groups=8, cross_attention_dim=16)
    torch.manual_seed(0)
    unet = UNet2DConditionModel(**cfg).eval()
    assert len(unet._resnets()) == 2 * 2 + 2 + 2 * 3            # down (2 x 2) + mid (2) + up (2 x 3)
    unet._batched_temb(torch.randn(1, 128))                     # fp32 CPU embedding: nothing is batched
    assert all(blk.temb_proj is None for blk in unet._resnets())


def test_conv2d_bias_residual_cpu_fallback_matches_conv2d():
    """ops.conv2d_bias_residual on CPU / fp32 is plain F.conv2d (+ residual); fold_bias drops the bias."""
    import torch
    from distrifuser_b200 import ops
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(8, 16, 3, padding=1)
    x, res = torch.randn(2, 8, 6, 5), torch.randn(2, 16, 6, 5)
    with torch.no_grad():
        ref = conv(x)
        assert torch.allclose(ops.conv2d_bias_residual(x, conv, conv.padding), ref)
        assert torch.allclose(ops.conv2d_bias_residual(x, conv, conv.padding, residual=res), ref + res)
        assert torch.allclose(ops.conv2d_bias_residual(x, conv, conv.padding, fold_bias=True), ref - conv.bias[None, :, None, None], atol=1e-6)
        other = torch.randn(16)
        assert torch.allclose(ops.conv2d_bias_residual(x, conv, conv.padding, bias=other), ref - conv.bias[None, :, None, None] + other[None, :, None, None], atol=1e-6)


def test_resnet_block_does_not_fold_biases_on_cpu():
    """The fused bias paths of compat.ResnetBlock2D are CUDA/fp16 only: on CPU the block is the textbook sequence."""
    import torch
    from distrifuser_b200.compat.unet_2d_condition import ResnetBlock2D
    torch.manual_seed(0)
    blk = ResnetBlock2D(32, 64, 16, 8, 1e-5)
    x, temb = torch.randn(1, 32, 6, 6), torch.randn(1, 16)
    assert not blk.folds_conv1_bias()
    with torch.no_grad():
        h = blk.conv1(torch.nn.functional.silu(blk.norm1(x)))
        h = h + blk.time_emb_proj(torch.nn.functional.silu(temb))[:, :, None, None]
        h = blk.conv2(torch.nn.functional.silu(blk.norm2(h)))
        ref = blk.conv_shortcut(x) + h
        assert torch.allclose(blk(x, temb), ref, atol=1e-5)
