import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle_libs():
    import uhdr_testlib as T
    T.ensure_oracle_built()
    return T


@pytest.fixture(scope="session")
def checker(oracle_libs):
    """The CPU implementation GPU results are compared with: the reference's own code when
    oracle/_ref was built, else the C restatement."""
    T = oracle_libs
    return T.Ref() if T.have_ref() else T.Oracle()


@pytest.fixture(scope="session")
def gpu():
    import torch
    import uhdr_testlib as T
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as g
    g.build()
    return T.Gpu()
