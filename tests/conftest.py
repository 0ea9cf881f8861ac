import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def oracle():
  from oracle import oracle as O
  O.lib()
  return O


@pytest.fixture(scope="session")
def ctx():
  """Process-wide GPU context.  GPU tests must fail (not skip) when the
  native path is unavailable: a silent fallback would void every parity claim."""
  from igneous_b200 import _shim
  return _shim.default_context()
