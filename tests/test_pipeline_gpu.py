"""End-to-end: DistriSDXLPipeline.__call__ (the reference's public API, pipelines.py:47-58) over a full denoising
trajectory -- warm-up synchronous steps, then displaced (1-step-stale) asynchronous steps, CFG, Euler -- against the same
trajectory computed with the oracle UNet path in fp32 on CPU.  The reference validates images with PSNR
(scripts/compute_metrics.py:62-79); on latents of a random-weight UNet we require PSNR > 35 dB (peak = max |ref|) after
6 steps, identical latent shapes, and bit-identical latents on every rank."""
import dataclasses

import pytest
import torch

from helpers import psnr
from oracle import harness, workloads
from mp_product import run_product_trajectory

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,graph", [("sdxl_w1", True), ("sdxl_w2_nosplit", True),
                                        ("sd15_w2_nosplit", True)])     # SD1.x: DistriSDPipeline.__call__, DDIM scheduler
def test_trajectory_matches_oracle(name, graph):
    case = dataclasses.replace({c.name: c for c in workloads.UNET_CASES}[name], warmup_steps=2)
    want = harness.run_trajectory(case, num_steps=6)
    got = run_product_trajectory(case, num_steps=6, use_graph=graph)
    for r, lat in enumerate(got):
        assert lat.shape == want.shape == (1, 4, case.latent, case.latent)
        assert torch.isfinite(lat).all()
        assert torch.equal(lat, got[0]), "every rank must hold the same latents"
        p = psnr(lat, want)
        assert p > 35.0, f"{name} rank{r}: PSNR {p:.1f} dB vs the fp32 oracle trajectory"


@pytest.mark.parametrize("family", ["sdxl", "sd15"])
def test_from_pretrained_with_diffusers_type_check(family):
    """Distri{SDXL,SD}Pipeline.from_pretrained (pipelines.py:20-42,179-200) against a `diffusers` whose pipeline
    constructor type-checks `unet=` against ModelMixin (as the real package does): BaseModel must derive from the mixins."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "run_from_pretrained.py"), family], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and "OK from_pretrained" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
