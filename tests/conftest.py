import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import refgold  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """Everything compiled: product library, oracle port, generator (and oracle/_ref when sources exist)."""
    import __graft_entry__ as ge
    ge.build()
    return True


@pytest.fixture(scope="session")
def ref(built):
    """The unmodified reference as a library, where oracle/_ref was built from its sources; None elsewhere (the parity tests
    then compare with the digests in tests/golden/reference_digests.json)."""
    from oracle import loaders
    if not os.path.exists(loaders.REFERENCE_SO):
        return None
    lib = loaders.load_reference()
    lib.set_verbose(0)
    return lib


@pytest.fixture(scope="session")
def port(built):
    """The oracle port (oracle/ma_oracle.c): builds the pre-states that the parity tests hand to the library under test."""
    from oracle import loaders
    lib = loaders.load_oracle_port()
    lib.set_verbose(0)
    return lib


@pytest.fixture(scope="session")
def prod(built, port):
    if refgold.RECORD:          # recording the reference's side runs without a GPU: the port stands in for the CUDA library
        return port
    from miniasm_b200 import capi
    lib = capi.load_product(strict=False)
    lib.set_verbose(0)
    return lib


@pytest.fixture(scope="session")
def gold_store():
    store = refgold.Store()
    yield store
    store.save()


@pytest.fixture
def gold(gold_store, request):
    return refgold.Checker(gold_store, request.node.nodeid)


@pytest.fixture(scope="session")
def paf_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("paf"))
