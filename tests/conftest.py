import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90)")
    config.addinivalue_line("markers", "slow: full-size CPU oracle checks (tens of seconds)")


def rel_l2(a, b):
    import torch
    from tests.golden.cases import Sampled
    if isinstance(b, Sampled):      # fixture stored as a sample of its elements: compare those elements
        a, b = b.take(a.detach()), b.values
    a = a.detach().double().cpu().reshape(-1)
    b = b.detach().double().cpu().reshape(-1)
    return float(torch.linalg.norm(a - b) / (torch.linalg.norm(b) + 1e-30))


@pytest.fixture(scope="session")
def have_cuda():
    import torch
    return torch.cuda.is_available()


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need a CUDA device and the built library: skip them cleanly elsewhere (a plain `pytest tests`
    on the CPU build box then runs the CPU suite only)."""
    import torch
    lib = os.path.join(ROOT, "audioldm2_b200", "libaldm_b200.so")
    if torch.cuda.is_available() and os.path.exists(lib):
        return
    why = "no CUDA device" if not torch.cuda.is_available() else "libaldm_b200.so not built"
    skip = pytest.mark.skip(reason=f"gpu test: {why}")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
