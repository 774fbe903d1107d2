import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture
def mv_device():
    """MV_Init on the device backend for one process (world size 1 loop-back, the
    reference's unit-test mode, Test/unittests/multiverso_env.h:9-29)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.init()
    yield mv
    mv.shutdown()
    mv.FLAGS.reset()
