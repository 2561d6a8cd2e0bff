import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, GOLD):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (pytest -m gpu)")
    # the CPU checkers (torch ops, the OpenMP C leaf) must not start more threads than the container's CPU quota:
    # 128 threads under a 16-CPU quota spend their time throttled at barriers
    from oracle.host import host_threads
    n = host_threads()
    os.environ.setdefault("OMP_NUM_THREADS", str(n))
    import torch
    torch.set_num_threads(n)


@pytest.fixture(scope="session")
def golden():
    """(arrays, meta) of the fixtures generated from the real reference (tests/golden/make_golden.py)."""
    arrays = np.load(os.path.join(GOLD, "ref_cpu.npz"))
    with open(os.path.join(GOLD, "ref_cpu_meta.json")) as f:
        meta = json.load(f)
    return arrays, meta


def fq_mismatch(y, y_ref, step=None, atol=1e-9):
    """Return (fraction of elements that differ beyond 1e-5 relative (+atol), max |diff| in units of `step`)."""
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    r = np.asarray(y_ref, dtype=np.float64).reshape(-1)
    tol = 1e-5 * np.maximum(np.abs(r), np.abs(y)) + atol
    bad = np.abs(y - r) > tol
    frac = float(bad.mean()) if y.size else 0.0
    if step is None or not bad.any():
        return frac, 0.0
    return frac, float((np.abs(y - r)[bad] / step).max())
