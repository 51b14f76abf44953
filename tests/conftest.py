import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "diffusers_stub")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100: pytest -m gpu)")
    config.addinivalue_line("markers", "multigpu(n): needs n CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        ngpu = 0
    for item in items:
        if "gpu" in item.keywords and ngpu == 0:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        m = item.get_closest_marker("multigpu")
        if m is not None and ngpu < m.args[0]:
            item.add_marker(pytest.mark.skip(reason=f"needs {m.args[0]} GPUs, have {ngpu}"))


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
