import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="session")
def pgs():
    import incubator_pegasus_b200 as p
    if not os.path.exists(p.LIB_PATH):  # a fresh checkout: the test session builds the library (the package itself never does)
        import shutil
        import subprocess
        if shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc"):
            subprocess.check_call(["bash", os.path.join(ROOT, "incubator_pegasus_b200", "build.sh")])
    p.lib()
    return p


@pytest.fixture(scope="session")
def engine(pgs):
    eng = pgs.Engine()
    yield eng
    eng.close()
