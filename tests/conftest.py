import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
  sys.path.insert(0, REPO)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def gen_dir():
  """Folder holding the generated CUDA filter libraries (built on demand; nvcc cross-compiles without a GPU)."""
  from rednose_b200.filters import ensure_generated
  from rednose_b200.filters.kinematic import KinematicKalman
  from rednose_b200.filters.live import LiveKalman
  d = ensure_generated(KinematicKalman)
  ensure_generated(LiveKalman)
  return d


@pytest.fixture(scope="session")
def oracle_dir():
  """Folder holding the CPU oracle libraries (oracle/_ref); rebuilt here when the reference is mounted."""
  from oracle import build_ref
  names = ["kinematic", "live", "compare"]
  if build_ref.reference_available():
    for n in names:
      build_ref.build(n)
  missing = [n for n in names if not os.path.exists(os.path.join(build_ref.OUT, f"lib{n}.so"))]
  if missing:
    pytest.skip(f"oracle/_ref not built for {missing} and the reference checkout is not present")
  return build_ref.OUT
