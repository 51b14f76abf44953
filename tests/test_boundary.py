"""CPU checks of the drop-in boundary: the C-ABI library builds, loads and exports every symbol the header declares;
the product package never touches the oracle; the Python API surface mirrors the reference's names."""
import ctypes
import inspect
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libpath():
    from distrifuser_b200 import build
    return build.build()


def test_header_symbols_exported(libpath):
    header = open(os.path.join(ROOT, "include", "distrifuser_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(df_[a-z_0-9]+)\s*\(", header)))
    assert len(declared) >= 15
    lib = ctypes.CDLL(libpath)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    from distrifuser_b200 import _lib
    assert sorted(_lib.EXPORTS) == declared


def test_library_is_sm90a_wgmma(libpath):
    sass = subprocess.run(["cuobjdump", "-sass", libpath], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA.64x128x16", "HGMMA.64x64x16", "UTMALDG", "SYNCS"):
        assert mnemonic in sass, f"{mnemonic} missing: the attention kernel is not a wgmma/TMA/mbarrier kernel"
    assert "HGMMA.64x256x16" in sass, "the GEMM must issue 64x256 warpgroup MMAs"
    assert "HMMA." not in sass, "legacy mma.sync tensor path in the library"


def test_error_channel(libpath):
    from distrifuser_b200 import _lib
    L = _lib.lib()
    assert L.df_version() == 2
    rc = L.df_step_begin(None, 7, None)          # argument validation happens before any CUDA call
    assert rc != 0 and b"df_step_begin" in L.df_last_error()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "distrifuser_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f"{f} imports the oracle"
                assert "/root/reference" not in text, f"{f} reads the reference tree"


def test_no_code_path_switches():
    """Environment variables may only observe the product (NVTX ranges, the flag-wait timeout, which library build to load)
    or pick the Linears on the hand-written GEMM; none selects another code path, launch or tuning constant.  The CUDA sources
    read no environment and take no tuning constant from a -D flag."""
    import ast
    allowed = {"DF_LIB_PATH", "DF_NVCC_FLAGS", "DF_NVTX", "DF_SPIN_TIMEOUT_S", "DF_LINEAR"}
    found = set()
    for dirpath, _, files in os.walk(os.path.join(ROOT, "distrifuser_b200")):
        for f in files:
            if f.endswith(".py"):
                tree = ast.parse(open(os.path.join(dirpath, f)).read())
                found |= {n.value for n in ast.walk(tree) if isinstance(n, ast.Constant) and isinstance(n.value, str)
                          and re.fullmatch(r"DF_[A-Z0-9_]+", n.value)}
    assert "DF_LINEAR" in found and found <= allowed, f"environment switches outside the allowed set: {sorted(found - allowed)}"
    csrc = os.path.join(ROOT, "distrifuser_b200", "csrc")
    for f in os.listdir(csrc):
        text = open(os.path.join(csrc, f)).read()
        assert "getenv(" not in text, f"{f} reads the environment"
        assert not re.search(r"#\s*ifndef\s+DF_", text), f"{f} takes a tuning constant from a -D flag"


def test_api_surface_matches_reference_names():
    from distrifuser_b200.models.distri_sdxl_unet_pp import DistriUNetPP
    from distrifuser_b200.modules.base_module import BaseModule
    from distrifuser_b200.modules.pp.attn import DistriCrossAttentionPP, DistriSelfAttentionPP
    from distrifuser_b200.modules.pp.conv2d import DistriConv2dPP
    from distrifuser_b200.modules.pp.groupnorm import DistriGroupNorm
    from distrifuser_b200.pipelines import DistriSDPipeline, DistriSDXLPipeline
    from distrifuser_b200.utils import DistriConfig, PatchParallelismCommManager
    sig = inspect.signature(DistriConfig.__init__)
    assert list(sig.parameters)[1:] == ["height", "width", "do_classifier_free_guidance", "split_batch", "warmup_steps",
                                        "comm_checkpoint", "mode", "use_cuda_graph", "parallelism", "split_scheme",
                                        "verbose"]                                       # utils.py:24-37
    assert sig.parameters["warmup_steps"].default == 4 and sig.parameters["comm_checkpoint"].default == 60
    assert sig.parameters["mode"].default == "corrected_async_gn"
    for cls in (DistriSDXLPipeline, DistriSDPipeline):
        for m in ("from_pretrained", "__call__", "set_progress_bar_config", "prepare"):
            assert hasattr(cls, m)
    for m in ("register_tensor", "create_buffer", "get_buffer_list", "communicate", "enqueue", "clear"):
        assert hasattr(PatchParallelismCommManager, m)                                 # utils.py:130-199
    fwd = list(inspect.signature(DistriUNetPP.forward).parameters)
    assert fwd[1:4] == ["sample", "timestep", "encoder_hidden_states"] and fwd[-2:] == ["return_dict", "record"]
    assert list(inspect.signature(DistriConv2dPP.__init__).parameters)[1:] == ["module", "distri_config", "is_first_layer"]
    for cls in (DistriGroupNorm, DistriSelfAttentionPP, DistriCrossAttentionPP):
        assert issubclass(cls, BaseModule)
        assert list(inspect.signature(cls.__init__).parameters)[1:] == ["module", "distri_config"]


def test_rank_math_matches_reference():
    """batch_idx / split_idx / n_device_per_batch (utils.py:68-75,98-109) against the oracle's restatement."""
    from oracle.workloads import DuckConfig
    from distrifuser_b200.utils import DistriConfig
    c = DistriConfig.__new__(DistriConfig)
    for world in (1, 2, 4, 8):
        for cfg_on in (True, False):
            for split in (True, False):
                for rank in range(world):
                    d = DuckConfig(world, rank, height=64, width=64, do_classifier_free_guidance=cfg_on, split_batch=split)
                    c.world_size, c.rank, c.do_classifier_free_guidance, c.split_batch = world, rank, cfg_on, split
                    c.n_device_per_batch = d.n_device_per_batch
                    assert c.batch_idx() == d.batch_idx() and c.split_idx() == d.split_idx()
                    grp = c.patch_group_ranks()
                    assert rank in grp and len(grp) == d.n_device_per_batch


def test_base_model_derives_from_diffusers_mixins_when_importable():
    """ADVICE r1: with diffusers importable BaseModel must be a (ModelMixin, ConfigMixin) like the reference's
    (distrifuser/models/base_model.py:8), otherwise StableDiffusionXLPipeline.from_pretrained(unet=...) rejects it."""
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, os.path.join(here, "run_from_pretrained.py"), "check-bases"], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0 and "OK bases" in r.stdout, r.stdout + r.stderr
