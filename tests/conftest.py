import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: test needs a CUDA (H100) device")


@pytest.fixture(scope="session")
def built():
  """Build the CUDA library and the C oracle once per session (nvcc/gcc; no GPU needed to build)."""
  import __graft_entry__ as g

  g.build()
  return True
