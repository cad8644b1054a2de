import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")
  config.addinivalue_line("markers", "multigpu: test needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
  try:
    import torch
    n_gpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
  except Exception:  # pragma: no cover
    n_gpu = 0
  skip_gpu = pytest.mark.skip(reason="needs a CUDA device")
  skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
  for item in items:
    if "gpu" in item.keywords and n_gpu == 0:
      item.add_marker(skip_gpu)
    if "multigpu" in item.keywords and n_gpu < 2:
      item.add_marker(skip_multi)
