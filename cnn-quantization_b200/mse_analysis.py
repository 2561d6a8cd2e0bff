"""The clipping analysis of the paper's eq. 6 (the reference's mse_analysis.py) in float64 torch: the analytic clipping +
quantization MSE of a Laplace(0, b) or Gauss(0, sigma) prior clipped to [-alpha, alpha] and quantized uniformly to
2^bit_width levels, and its simulation on a given sample.

    mse_laplace(alpha) = 2 b^2 exp(-alpha / b) + alpha^2 / (3 * 4^bits)
    mse_gaus(alpha)    = (sigma^2 + alpha^2) (1 - erf(alpha / (sigma sqrt 2))) - sqrt(2 / pi) alpha sigma exp(-alpha^2 / (2 sigma^2))
                         + alpha^2 / (3 * 4^bits)

The simulations take the sample as an argument instead of drawing it; everything else follows the reference's
operations.  ``collect_mse`` (statistics.ClipMseStatistics) puts the analytic curves beside the measured ones.

Run as a script, the module writes the reference's two curves (simulation and analysis over alpha = 5, 5.1, ..., 19.9 at
4 bits, b or sigma = 2, 100 000 samples) as CSV instead of plotting them:

    python -m cnn_quantization_b200.mse_analysis [--prior laplace|gaus] [--seed N] [--out curves.csv]
"""
import argparse
import math
import sys

import numpy as np
import torch

__all__ = ["uniform_midtread_quantizer", "LaplacianClippingAnalysis", "GaussianClippingAnalysis",
           "LaplacianClippingSimulation", "GaussianClippingSimulation"]


def _f64(v):
    return torch.as_tensor(v, dtype=torch.float64)


def uniform_midtread_quantizer(x, Q):
    """round(x / Q) * Q, rounding half to even as numpy does."""
    return torch.round(x / Q) * Q


def LaplacianClippingAnalysis(Alpha, b, bitWidth):
    """Analytic MSE of Laplace(0, b) data clipped at each alpha of ``Alpha``, float64 tensor."""
    alpha = _f64(Alpha)
    return 2 * (b ** 2) * torch.pow(_f64(math.e), -alpha / b) + (alpha * alpha) / (3 * (2 ** (2 * bitWidth)))


def GaussianClippingAnalysis(Alpha, sigma, bitWidth):
    """Analytic MSE of Gauss(0, sigma) data clipped at each alpha of ``Alpha``, float64 tensor."""
    alpha = _f64(Alpha)
    a2 = alpha * alpha
    clipping = ((sigma ** 2 + a2) * (1 - torch.erf(alpha / (sigma * math.sqrt(2.0))))
                - math.sqrt(2.0 / math.pi) * alpha * sigma * torch.pow(_f64(math.e), ((-1) * (0.5 * a2)) / sigma ** 2))
    return clipping + a2 / (3 * (2 ** (2 * bitWidth)))


def _clipping_simulation(Alpha, sample, bitWidth):
    x = _f64(sample)
    out = []
    for alpha in _f64(Alpha).tolist():
        Q = (2 * alpha) / (2 ** bitWidth)
        s = uniform_midtread_quantizer(torch.clamp(x, -alpha, alpha), Q)
        out.append(((s - x) ** 2).mean())
    return torch.stack(out) if out else torch.zeros(0, dtype=torch.float64)


def LaplacianClippingSimulation(Alpha, sample, bitWidth):
    """Measured MSE of ``sample`` (the reference draws np.random.laplace(scale=b, size=100000)) clipped at each alpha and
    quantized mid-tread with step 2 alpha / 2^bitWidth."""
    return _clipping_simulation(Alpha, sample, bitWidth)


def GaussianClippingSimulation(Alpha, sample, bitWidth):
    """Measured MSE of ``sample`` (the reference draws np.random.normal(0, sigma, size=100000)), as the Laplace one."""
    return _clipping_simulation(Alpha, sample, bitWidth)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--prior", choices=("laplace", "gaus"), default="laplace")
    ap.add_argument("--seed", type=int, default=None, help="np.random.seed before the sample is drawn")
    ap.add_argument("--out", default=None, help="CSV path (default: standard output)")
    a = ap.parse_args(argv)
    Alpha = np.arange(5, 20, 0.1)
    bitWidth, scale = 4, 2
    if a.seed is not None:
        np.random.seed(a.seed)
    if a.prior == "laplace":
        sim = LaplacianClippingSimulation(Alpha, np.random.laplace(scale=scale, size=100000, loc=0), bitWidth)
        ana = LaplacianClippingAnalysis(Alpha, scale, bitWidth)
    else:
        sim = GaussianClippingSimulation(Alpha, np.random.normal(0, scale, size=100000), bitWidth)
        ana = GaussianClippingAnalysis(Alpha, scale, bitWidth)
    f = open(a.out, "w") if a.out else sys.stdout
    try:
        f.write("alpha,simulation,analysis\n")
        for al, s, an in zip(Alpha.tolist(), sim.tolist(), ana.tolist()):
            f.write("%r,%r,%r\n" % (al, s, an))
    finally:
        if a.out:
            f.close()


if __name__ == "__main__":
    main()
