import os
import sys

import pytest

# VirtualCluster tests run up to 8 mutually-waiting kernels on 8 streams of one GPU: give every
# stream its own hardware queue so none is serialised behind a spinning peer (default is 8 queues).
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100)")
    config.addinivalue_line("markers", "multigpu: test needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    import torch

    has_gpu = torch.cuda.is_available()
    ngpu = torch.cuda.device_count() if has_gpu else 0
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
