import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    # the suites load the in-tree liblzgpu.so (host maths and ABI tests need it even without a GPU): build it if a fresh
    # checkout has not run __graft_entry__.build() yet (nvcc cross-compiles for sm_90a without a device)
    if not os.path.exists(os.path.join(ROOT, "lizardfs_b200", "liblzgpu.so")):
        import subprocess
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "lizardfs_b200", "csrc"), "-j8"], check=False)


@pytest.fixture(scope="session")
def oracle():
    from tests import _oracle
    return _oracle.load_oracle()


@pytest.fixture(scope="session")
def ref():
    """The UNMODIFIED reference compiled into oracle/_ref/liblzref.so (None when absent)."""
    from tests import _oracle
    return _oracle.load_ref()
