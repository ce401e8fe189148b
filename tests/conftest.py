import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def synth_mod():
    import synth
    synth.build_lib()
    return synth


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle
    oracle.build_lib()
    return oracle


@pytest.fixture(scope="session")
def ts1(synth_mod):
    return synth_mod.Tipset(synth_mod.config_params(1))


@pytest.fixture(scope="session")
def ts2(synth_mod):
    return synth_mod.Tipset(synth_mod.config_params(2))


@pytest.fixture(scope="session")
def ts3_small(synth_mod):
    return synth_mod.Tipset(synth_mod.config_params(3, hamt_entries=20000))


@pytest.fixture(scope="session")
def api():
    from ipc_filecoin_proofs_b200 import api as a
    a.lib()
    return a
