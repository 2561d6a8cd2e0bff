#!/usr/bin/env python
"""Synthetic bit-allocation fixture from the REAL reference's bit_allocation_synthetic.py (build container only), written
to ref_bit_alloc.npz.

The reference module imports matplotlib.pyplot at the top and only plots under ``__main__``: a stub module stands in
for it.  The three channel pairs of its ``__main__`` (sigma^(2/3) ratios 2:1, 1:2, 1:1; 2 000 samples each, drawn after
a fixed seed) are stored in the file, with the reference's own ``simulator3`` curves over its share range and one
``simulator`` call per sample.

    python tests/golden/make_bit_alloc_golden.py
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("FQB200_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "ref_bit_alloc.npz")

SEED = 21
SIGMAS = ((2.82845653294, 1.0), (1.0, 2.82845653294), (1.0, 1.0))
N = 2000      # 10 000 in the reference; fewer keeps the fixture small
Q = 32.0
SIM_STEP = 0.37   # the step of the single simulator() calls


def main():
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
    sys.path.insert(0, REF)
    ref = importlib.import_module("bit_allocation_synthetic")
    Range = list(ref.frange(0.15, 0.85, 0.01))
    np.random.seed(SEED)
    out = {"range": np.asarray(Range, dtype=np.float64)}
    for i, (sa, sb) in enumerate(SIGMAS):
        X = np.random.normal(0, sa, N)
        Y = np.random.normal(0, sb, N)
        sims, mse = ref.simulator3(X, Y, Q=Q, Range=Range)
        out["x%d" % i], out["y%d" % i] = X, Y
        out["simulations%d" % i] = np.asarray(sims, dtype=np.float64)
        out["mse%d" % i] = np.asarray(mse, dtype=np.float64)
        out["single%d" % i] = np.asarray(ref.simulator(X, SIM_STEP), dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
