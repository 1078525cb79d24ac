import os, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")
    config.addinivalue_line("markers", "multigpu: needs two or more CUDA devices on one box; run with -m multigpu")


def pytest_collection_modifyitems(config, items):
    # gpu tests must never silently pass without a GPU: they are skipped only when no CUDA device exists AND
    # the run did not ask for them (-m gpu on a GPU-less box fails loudly in the fixture below).
    pass


@pytest.fixture(scope="session")
def cuda():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test ran without a CUDA device"
    return torch.device("cuda:0")


GOLDEN = os.path.join(ROOT, "tests", "golden")
