"""pytest configuration: registers the ``gpu`` marker and puts the repo root on sys.path.

``-m "not gpu"`` tests: the oracle against the reference's golden vectors, host logic, C-ABI symbol
checks.  ``-m gpu`` tests: parity of the CUDA path (through the C-ABI) against the oracle.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the library is built for sm_90a)")


def _load_pkg():
    import __graft_entry__ as ge
    if not os.path.exists(os.path.join(ge.PKG_DIR, "libbydbgpu.so")):
        ge.build()  # a fresh checkout has no built artefacts (they are git-ignored): compile the CUDA library first
    return ge.load_package()


import pytest  # noqa: E402


@pytest.fixture(scope="session")
def bydb():
    """The product package (skywalking-banyandb_b200/) under its import name bydb_b200."""
    return _load_pkg()


@pytest.fixture(scope="session")
def gpu_ctx(bydb):
    ctx = bydb.Context(device=0)
    yield ctx
    ctx.close()
