import os
import sys

import pytest

os.environ.setdefault("DDS_COMM_TIMEOUT_S", "40")  # a wedged rank should fail a test in seconds, not minutes
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _ensure_built():
    """the native pieces are built in-tree by __graft_entry__.build(); build now if this checkout has not been built
    yet (fresh clone: *.so is git-ignored) or if a source is newer than the library it goes into"""
    import glob
    lib = os.path.join(ROOT, "ddstore_b200", "libddstore_b200.so")
    cy = glob.glob(os.path.join(ROOT, "ddstore_b200", "cython", "pyddstore*.so"))
    orc = os.path.join(ROOT, "oracle", "liboracle.so")
    stale = not os.path.exists(lib) or not cy or not os.path.exists(orc)
    if not stale:
        srcs = glob.glob(os.path.join(ROOT, "ddstore_b200", "csrc", "*.c*")) + \
            glob.glob(os.path.join(ROOT, "ddstore_b200", "csrc", "*.h")) + glob.glob(os.path.join(ROOT, "include", "*.h*"))
        stale = max(os.path.getmtime(f) for f in srcs) > os.path.getmtime(lib) or \
            os.path.getmtime(os.path.join(ROOT, "ddstore_b200", "cython", "pyddstore.pyx")) > os.path.getmtime(cy[0]) or \
            os.path.getmtime(os.path.join(ROOT, "oracle", "ddstore_oracle.c")) > os.path.getmtime(orc)
    if stale:
        import __graft_entry__
        __graft_entry__.build()


def pytest_configure(config):
    _ensure_built()
    config.addinivalue_line("markers", "gpu: needs an H100 GPU")
    config.addinivalue_line("markers", "multigpu: needs >= 2 GPUs on the box")


@pytest.fixture(scope="session")
def coracle():
    from oracle.oracle import COracle
    return COracle()
