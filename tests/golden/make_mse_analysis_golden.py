#!/usr/bin/env python
"""Clipping-analysis fixture (eq. 6 of the paper) from the REAL reference's mse_analysis.py (build container only),
written to ref_mse_analysis.npz.

The reference module imports matplotlib.pyplot at the top and only plots under ``__main__``: a stub module stands in
for it.  Each case seeds ``np.random`` and calls the reference's own Laplacian / Gaussian ClippingAnalysis and
ClippingSimulation; the simulations draw their 100 000-sample input inside, right after the seed, so the test redraws
the same sample from the recorded seed (numpy's legacy RandomState stream is fixed) and feeds it to the port.  The
sample's sum is recorded to catch a different stream.

    python tests/golden/make_mse_analysis_golden.py
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("FQB200_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "ref_mse_analysis.npz")

# (name, prior, Alpha, scale (b or sigma), bitWidth, seed): the reference's own __main__ settings first
CASES = [
    ("laplace_main", "laplace", np.arange(5, 20, 0.1), 2, 4, 11),
    ("gaus_main", "gaus", np.arange(5, 20, 0.1), 2, 4, 12),
    ("laplace_2bit", "laplace", np.arange(0.25, 8, 0.125), 1.5, 2, 13),
    ("gaus_8bit", "gaus", np.arange(0.5, 12, 0.25), 0.75, 8, 14),
]


def draw(prior, scale, seed):
    """The sample the reference's simulation draws right after np.random.seed(seed)."""
    np.random.seed(seed)
    if prior == "laplace":
        return np.random.laplace(scale=scale, size=100000, loc=0)
    return np.random.normal(0, scale, size=100000)


def main():
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
    sys.path.insert(0, REF)
    ref = importlib.import_module("mse_analysis")
    out = {}
    for name, prior, Alpha, scale, bits, seed in CASES:
        np.random.seed(seed)
        if prior == "laplace":
            sim = ref.LaplacianClippingSimulation(Alpha, scale, bits)
            ana = ref.LaplacianClippingAnalysis(Alpha, scale, bits)
        else:
            sim = ref.GaussianClippingSimulation(Alpha, scale, bits)
            ana = ref.GaussianClippingAnalysis(Alpha, scale, bits)
        out[name + "_alpha"] = Alpha
        out[name + "_meta"] = np.array([scale, bits, seed, draw(prior, scale, seed).sum()], dtype=np.float64)
        out[name + "_simulation"] = np.asarray(sim, dtype=np.float64)
        out[name + "_analysis"] = np.asarray(ana, dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
