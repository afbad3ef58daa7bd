import os
import sys

import pytest

# several ranks' plans share one GPU in the transport tests: give every stream its own hardware queue, otherwise a
# spinning wait kernel can sit in front of the very put kernel it waits for (false dependency through a shared queue)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
# (the library preloads its own kernels when peers are wired: a lazy load synchronises with the device, i.e. with the
# spinning wait kernel of the rank that waits for the very launch being loaded; CUDA_MODULE_LOADING=EAGER would do the
# same but makes every process load all of torch's kernels — minutes)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def golden_cases():
    return ["gemat11_k1", "gemat11_k2", "gemat11_k3_hp", "gemat11_k3_rp", "karate_k3_hp", "karate_k3_stchp"]


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
