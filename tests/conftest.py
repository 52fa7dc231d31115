import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# keep every test hermetic: private BEE2BEE_HOME, no WAN probing
os.environ.setdefault("BEE2BEE_OFFLINE", "1")
# no network -> no checkpoints: the suites run the real architectures on random-init weights (opt-in, see
# models/weights.py::random_weights_allowed; test_weights_policy covers the default refusal)
os.environ.setdefault("B2B_ALLOW_RANDOM_WEIGHTS", "1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "timeout(seconds): per-test limit (pytest-timeout; inert without the plugin)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _isolated_home(tmp_path, monkeypatch):
    monkeypatch.setenv("BEE2BEE_HOME", str(tmp_path / "b2b_home"))
    yield
