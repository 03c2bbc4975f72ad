import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def po():
    """The CPU oracle (test infrastructure)."""
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def goldens():
    import json
    return json.load(open(os.path.join(ROOT, "tests", "golden", "reference_goldens.json"), encoding="utf-8"))


@pytest.fixture(scope="session")
def eng():
    """One engine on cuda:0. Fails loudly when the CUDA library is missing: there is no CPU fallback."""
    from transferia_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()
