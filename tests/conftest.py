import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_cuda = torch.cuda.is_available()
        ngpu = torch.cuda.device_count() if has_cuda else 0
    except Exception:  # pragma: no cover
        has_cuda, ngpu = False, 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and not has_cuda:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(skip_multi)


@pytest.fixture
def tmp_ckpt(tmp_path):
    return str(tmp_path / "test.pth")


@pytest.fixture
def legacy_conv_schedule(monkeypatch):
    """The round-1 ResNet step schedule (every entry of fl.convnet.SCHEDULE_DEFAULTS at 0).  Tests that switch ONE
    re-scheduling on and compare it with "the base" were written against that base; the shipped defaults (the fastest
    measured combination) are covered by the tests that do not use this fixture."""
    from colearn_federated_learning_b200.fl import convnet
    for k in list(convnet.SCHEDULE_DEFAULTS):
        monkeypatch.setitem(convnet.SCHEDULE_DEFAULTS, k, 0)
    for k in list(os.environ):
        if k.startswith("COLEARN_CONV_"):
            monkeypatch.delenv(k, raising=False)
