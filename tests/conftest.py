import os
import sys

# The CPU oracle runs torch's OpenMP kernels.  With the default ACTIVE wait policy idle OpenMP threads spin, and on a host whose
# cores are shared with other jobs that spinning collapses throughput (measured in the build container: the same six oracle
# tests take 6 s alone, 136 s with three copies running side by side, 15 s with OMP_WAIT_POLICY=PASSIVE).  Must be set before
# torch (libgomp) is loaded; a caller's own setting wins.
os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")

import pytest  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(autouse=True, scope="session")
def _bounded_cpu_threads():
    """The CPU oracle (torch convolutions on 64x64 images) is fastest with 8-16 intra-op threads and collapses on the 100+
    cores of a GPU box; every test that runs it gets a bounded pool."""
    import torch

    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))
    yield
