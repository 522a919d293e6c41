import os, sys
import pytest

# The checker (oracle/_ref: the reference's C++/OpenMP) and torch bring two OpenMP runtimes into the test process; on a
# many-core box their spin-waiting worker pools starve each other (a 2 s oracle call took > 60 s on 128 cores).
os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")
os.environ.setdefault("OMP_NUM_THREADS", "8")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box with `pytest -m gpu`)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
