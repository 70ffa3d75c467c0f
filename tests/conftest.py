import os
import sys

import pytest

# simulated multi-rank worlds put up to 8 spinning kernels on 8 streams of one
# GPU: give every stream its own hardware queue (must precede CUDA init).
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100)")
    config.addinivalue_line("markers", "multigpu: test needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
        ngpu = torch.cuda.device_count() if has_gpu else 0
    except Exception:  # pragma: no cover
        has_gpu, ngpu = False, 0
    skip_gpu = pytest.mark.skip(reason="needs a CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(skip_multi)


@pytest.fixture(autouse=True)
def _clean_parallax_env(monkeypatch):
    for k in list(os.environ):
        if k.startswith("PARALLAX_") and k not in ("PARALLAX_LOG_LEVEL",):
            monkeypatch.delenv(k, raising=False)
    import parallax_b200.shard as sh
    sh.reset()
    yield
