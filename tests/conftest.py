"""Test configuration.

* ``-m "not gpu"``: oracle vs golden vectors, host logic, C-ABI symbol export — runs anywhere.
* ``-m gpu``: parity tests proper, through the C ABI on a real H100.

The oracle (``oracle/``) is imported here and in the test modules only as the checker.
"""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """Native library + C oracle built in-tree (nvcc cross-compiles without a GPU)."""
    from learningorchestra_b200.build import build_all
    build_all()
    return True


@pytest.fixture(scope="session")
def engine(built):
    from learningorchestra_b200.engine import Engine
    eng = Engine(0)          # raises LoexecError without an H100: gpu tests must not silently pass
    yield eng
    eng.close()
