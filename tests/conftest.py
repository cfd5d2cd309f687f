import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

# The oracle configures PYTENSOR_FLAGS (compile dir, BLAS for the reference C linker) before pytensor is imported.
from oracle import cvm as _cvm  # noqa: E402

_cvm.configure()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu():
    if os.environ.get("PTK_DRY") == "1":
        return False  # developer dry run on a CPU box: lower every graph, run only the reference
    if not has_gpu():
        pytest.skip("no CUDA device")
    import pytensor_b200  # noqa: F401
    from pytensor_b200.runtime import device

    device.device()
    return True
