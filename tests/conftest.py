import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu)")


@pytest.fixture(scope="session")
def hierarchy():
    from cape_b200 import topology as T
    L, D, U, p, L_d, D_d, U_d = T.load_graph_mtx(load_for_demo=True)
    return dict(L=L, D=D, U=U, p=p, L_d=L_d, D_d=D_d, U_d=U_d)


@pytest.fixture(scope="session")
def lib_built():
    """Build libcape_b200.so if it is missing (nvcc cross-compiles without a GPU)."""
    from cape_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()
