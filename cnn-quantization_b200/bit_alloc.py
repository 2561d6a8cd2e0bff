"""Per-channel bit allocation from measured errors (`-bap mse`), and the reference's synthetic bit-allocation experiment
(bit_allocation_synthetic.py) in float64 torch.

``allocate(sse, target)`` takes a [G, 9] table whose entry [g, w] is the error channel g's quantizer makes at w bits
(ops.clip_mse with widths 0..8) and returns the widths that minimise the total error for the budget of ``target`` bits
per channel on average:

    minimise  sum_g sse[g, w_g]   subject to   sum_g w_g <= floor(target * G),   w_g in 0..8

It is an exact dynamic programme over (channel, bits left), run from the last channel to the first in float64 on the
host, with a uint8 choice table.  Among minimisers it returns the lexicographically smallest width vector (channel 0
first): each channel takes the smallest width that reaches the optimum of what is left, so a channel whose errors are
equal at every width (a constant channel) gets 0 bits.  At G = 2048 and target 4 it makes about 2048 x 8193 x 9 updates
(nine vector operations of 8193 entries per channel) and a 16 MB choice table.

``simulator`` and ``simulator3`` are the reference's two-channel Gaussian experiment with the samples as arguments, like
mse_analysis.py.  Run as a script, the module writes the reference's three curves (the MSE of two channels sharing 32
bins, over the share p of channel X, for alpha^(2/3) ratios 2:1, 1:2 and 1:1) as CSV instead of plotting them:

    python -m cnn_quantization_b200.bit_alloc [--seed N] [--out curves.csv]
"""
import argparse
import math
import sys

import numpy as np
import torch

__all__ = ["MAX_BITS", "allocate", "frange", "uniform_midtread_quantizer", "simulator", "simulator3"]

MAX_BITS = 8


def allocate(sse, target):
    """int64 [G] widths in 0..8 minimising sum_g sse[g, w_g] with sum_g w_g <= floor(target * G); ties go to the
    lexicographically smallest width vector.  ``sse``: [G, 9] finite values (numpy or torch, used as float64)."""
    if isinstance(sse, torch.Tensor):
        sse = sse.detach().cpu().numpy()
    e = np.asarray(sse, dtype=np.float64)
    if e.ndim != 2 or e.shape[1] != MAX_BITS + 1 or e.shape[0] < 1:
        raise ValueError("allocate needs a [G, %d] error table, got shape %s" % (MAX_BITS + 1, e.shape))
    if not np.isfinite(e).all():
        raise ValueError("allocate needs finite errors")
    g = e.shape[0]
    budget = min(int(math.floor(target * g)), MAX_BITS * g)
    if budget < 0:
        raise ValueError("allocate: target %r gives a negative budget" % (target,))
    # best[b] = least error of the channels after the current one with at most b bits; choice[c, b] = channel c's width
    best = np.zeros(budget + 1)
    choice = np.zeros((g, budget + 1), dtype=np.uint8)
    for c in range(g - 1, -1, -1):
        new = np.full(budget + 1, np.inf)
        pick = choice[c]
        for w in range(min(MAX_BITS, budget) + 1):
            cand = e[c, w] + best[:budget + 1 - w]
            better = cand < new[w:]   # strict: a tie keeps the smaller width
            new[w:][better] = cand[better]
            pick[w:][better] = w
        best = new
    widths = np.empty(g, dtype=np.int64)
    b = budget
    for c in range(g):
        widths[c] = choice[c, b]
        b -= int(widths[c])
    return widths


# ---- bit_allocation_synthetic.py -------------------------------------------------------------------------------------------
def frange(x, y, jump):
    """x, x + jump, ... while < y, accumulated as the reference does."""
    while x < y:
        yield x
        x += jump


def uniform_midtread_quantizer(x, Q):
    """round(x / Q) * Q, rounding half to even as numpy does."""
    return torch.round(x / Q) * Q


def simulator(Val, Q):
    """[MSE of ``Val`` quantized mid-tread with step Q, Q], float64."""
    v = torch.as_tensor(Val, dtype=torch.float64)
    s = uniform_midtread_quantizer(v.clone(), Q)
    return [((s - v) ** 2).mean(), Q]


def simulator3(X, Y, Q, Range):
    """[simulations, MSE] of two channels X and Y sharing Q bins: for each share p of ``Range``, X gets p * Q bins over its
    range and Y (1 - p) * Q; both lists hold mse_X + mse_Y as float64 scalars."""
    x = torch.as_tensor(X, dtype=torch.float64)
    y = torch.as_tensor(Y, dtype=torch.float64)
    simulations, MSE = [], []
    for p in Range:
        Delta_X = float(x.max() - x.min()) / (p * Q)
        Delta_Y = float(y.max() - y.min()) / ((1 - p) * Q)
        mse_X = simulator(x, Delta_X)[0]
        mse_Y = simulator(y, Delta_Y)[0]
        simulations.append(mse_X + mse_Y)
        MSE.append(mse_X + mse_Y)
    return [simulations, MSE]


# the reference's three channel pairs: sigma^(2/3) ratios 2:1, 1:2 and 1:1
SIGMAS = ((2.82845653294, 1.0), (1.0, 2.82845653294), (1.0, 1.0))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--seed", type=int, default=None, help="np.random.seed before the samples are drawn")
    ap.add_argument("--out", default=None, help="CSV path (default: standard output)")
    a = ap.parse_args(argv)
    Range = list(frange(0.15, 0.85, 0.01))
    n = 10000
    if a.seed is not None:
        np.random.seed(a.seed)
    samples = [(np.random.normal(0, sa, n), np.random.normal(0, sb, n)) for sa, sb in SIGMAS]
    curves = [simulator3(X, Y, Q=32.0, Range=Range)[1] for X, Y in samples]
    f = open(a.out, "w") if a.out else sys.stdout
    try:
        f.write("p,mse_a,mse_b,mse_c\n")
        for i, p in enumerate(Range):
            f.write("%r,%r,%r,%r\n" % (p, float(curves[0][i]), float(curves[1][i]), float(curves[2][i])))
    finally:
        if a.out:
            f.close()


if __name__ == "__main__":
    main()
