import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


def pytest_sessionstart(session):
    """Build artefacts are git-ignored: bring them up to date (nvcc cross-compiles without a GPU).  make rebuilds what is
    missing or stale (e.g. objects from an older Makefile's architecture flags) and does nothing otherwise."""
    import subprocess
    subprocess.check_call(['make', '-C', os.path.join(ROOT, 'circom_compat_b200', 'csrc'), '-j4'], stdout=subprocess.DEVNULL)
    subprocess.check_call(['make', '-C', os.path.join(ROOT, 'oracle')], stdout=subprocess.DEVNULL)


@pytest.fixture(scope='session')
def golden():
    return json.load(open(os.path.join(GOLDEN, 'golden_vectors.json')))


@pytest.fixture(scope='session')
def test_zkey_bytes():
    return open(os.path.join(GOLDEN, 'test.zkey'), 'rb').read()


@pytest.fixture(scope='session')
def complex_zkey_bytes():
    return open(os.path.join(GOLDEN, 'complex-circuit-10000-10000.zkey'), 'rb').read()


@pytest.fixture(scope='session')
def ctx():
    """A real device context.  GPU tests never skip and never fall back: no CUDA => failure."""
    from circom_compat_b200 import Context
    from circom_compat_b200 import release_all
    c = Context(0)
    yield c
    release_all()
    c.close()
