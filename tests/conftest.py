"""pytest configuration: registers the ``gpu`` marker and shared fixtures.

``-m "not gpu"`` runs without a GPU; ``-m gpu`` runs on an H100.  Both use only committed fixtures.
"""
import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def golden_names(prefix="msda_"):
    return sorted(os.path.basename(p)[len(prefix):-4]
                  for p in glob.glob(os.path.join(GOLDEN_DIR, prefix + "*.npz")))


def load_golden(name, prefix="msda_"):
    with np.load(os.path.join(GOLDEN_DIR, f"{prefix}{name}.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
