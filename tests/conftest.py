import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90); run with -m gpu on a machine that has one")
    # The built library is git-ignored: a fresh checkout has none.  Build it (nvcc cross-compiles without a GPU) rather than fail every
    # test at import; where nvcc is missing too the tests fail loudly in _lib.load(), as the product does.
    lib = os.path.join(ROOT, "bundletrack_b200", "lib", "libbundletrack_b200.so")
    if not os.path.exists(lib):
        import shutil
        import subprocess
        if shutil.which("nvcc") and shutil.which("make"):
            subprocess.call(["make", "-C", os.path.join(ROOT, "bundletrack_b200", "csrc"), "-j8"])


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
