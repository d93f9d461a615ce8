import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `-m gpu`)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 GPUs on the box")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        have_gpu = torch.cuda.is_available()
        ngpu = torch.cuda.device_count() if have_gpu else 0
    except Exception:
        have_gpu, ngpu = False, 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 GPUs")
    for item in items:
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(skip_multi)


@pytest.fixture
def fresh_flags():
    from distributedmnist_b200.flags import FLAGS
    FLAGS.reset()
    yield FLAGS
    FLAGS.reset()
