import atexit
import os
import shutil
import sys
import tarfile
import tempfile
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _unpack_reference_data():
    """The original project's data files the tests compare against (tests/golden/make_reference_data.py), unpacked with
    the layout of an IsaacGymEnvs checkout into a directory removed when the session ends.  The original task modules that
    build() staged under oracle/_ref/ (oracle/ref_tasks.py) are laid over it."""
    d = tempfile.mkdtemp(prefix="igedata_")
    atexit.register(shutil.rmtree, d, True)
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "reference_data.tar.xz")) as tar:
        tar.extractall(d, filter="data")
    staged = os.path.join(ROOT, "oracle", "_ref")
    if os.path.isdir(os.path.join(staged, "isaacgymenvs")):
        shutil.copytree(staged, d, dirs_exist_ok=True)
    return d


REFERENCE = _unpack_reference_data()
# The tests that run the original task modules on the compat shim: an IsaacGymEnvs checkout, or the tree above when build()
# staged the modules.
CHECKOUT = os.environ.get("ISAACGYMENVS_ROOT", "") or REFERENCE
needs_checkout = pytest.mark.skipif(not os.path.isdir(os.path.join(CHECKOUT, "isaacgymenvs", "tasks")),
                                    reason="no IsaacGymEnvs task modules: build() found no checkout to stage them from")
