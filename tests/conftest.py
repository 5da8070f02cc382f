import os
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
# the trainers' `datasets` pipeline writes a cache (HF_HOME / HF_DATASETS_CACHE, by default under ~/.cache/huggingface); the
# suite may run as a user whose home is not writable, so it always gets a cache of its own (inherited by the CLI subprocesses)
_HF = os.path.join(tempfile.gettempdir(), f"dalm_b200_tests_hf_{os.getuid()}")
os.environ["HF_HOME"] = _HF
os.environ["HF_DATASETS_CACHE"] = os.path.join(_HF, "datasets")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def cuda_dev():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from dalm_b200 import _lib

    _lib.call("dalm_b200_probe_device")
    return torch.device("cuda:0")
