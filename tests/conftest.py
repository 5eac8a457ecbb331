import os
import sys

# Several ranks of the slab engine may share one device in these tests (a one-GPU box still runs
# the whole exchange).  Their pull kernels spin until a peer's push kernel has run, so kernels of
# different streams must really be able to run side by side: with more streams than hardware
# work queues (default 8) two streams can share a queue and a spinning kernel would then sit in
# front of the very kernel it waits for.  Must be set before CUDA initialises.  Production runs
# one rank per device and never needs it.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "needs_ref: needs oracle/_ref built from /root/reference")


@pytest.fixture(scope="session", autouse=True)
def _build_test_infra():
    """Build the oracle restatement / fake libjpeg front end if missing (gcc only)."""
    import oracle_lib
    oracle_lib.ensure_built()
    yield
