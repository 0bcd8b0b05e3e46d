import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _ensure_built():
    """A fresh clone has no binaries (they are git-ignored): build the library if it is missing."""
    import subprocess
    lib = os.path.join(ROOT, "soilmachine_b200", "lib", "libsoilmachine_b200.so")
    if not os.path.exists(lib):
        subprocess.check_call(["bash", os.path.join(ROOT, "build.sh")])


_ensure_built()


@pytest.fixture(scope="session")
def ref():
    """The reference's own hot path (oracle/_ref/libsmref.so)."""
    from oracle import refapi
    if not refapi.available():
        pytest.skip("oracle/_ref/libsmref.so not built (make -C oracle ref)")
    return refapi.get()
