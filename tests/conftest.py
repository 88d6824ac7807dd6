"""pytest configuration: markers + import plumbing.

`-m "not gpu"` = oracle vs the reference's golden vectors, host logic, C-ABI symbol
checks (runs anywhere).  `-m gpu` = parity tests proper: the CUDA path called through
the C-ABI vs the oracle (needs an H100).
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_sessionstart(session):
    """Built artefacts are git-ignored.  With nvcc present the incremental build (mtime-gated, cheap when nothing
    changed) always runs, so the tests never see a stale library; without nvcc only the CPU oracle is built (make) and
    the product-library tests fail or skip individually instead of aborting the whole session."""
    import shutil
    import subprocess

    import __graft_entry__ as ge

    have_nvcc = bool(shutil.which("nvcc")) or os.path.exists("/usr/local/cuda/bin/nvcc")
    if have_nvcc:
        ge.build()
    else:
        try:
            ge.build_oracle()
        except (subprocess.CalledProcessError, OSError):
            pass


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o

    o.lib()
    return o


@pytest.fixture(scope="session")
def kb():
    """The product package (loads libkornia_b200.so; fails loudly if it is missing)."""
    import kornia_rs_b200

    return kornia_rs_b200
