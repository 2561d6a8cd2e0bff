"""Deterministic inputs for the golden fixtures (numpy RandomState: stable across numpy versions).

Shared by the fixture generators (which need the reference, or its compiled extension and a GPU) and by the tests.
"""
import numpy as np


def make_input(seed, shape, dist="normal", relu=False, chan_scale=True):
    rs = np.random.RandomState(seed)
    if dist == "normal":
        x = rs.standard_normal(shape)
    elif dist == "laplace":
        x = rs.laplace(size=shape)
    else:
        raise ValueError(dist)
    if chan_scale and len(shape) >= 2:
        cdim = 1 if len(shape) == 4 else 0
        sc = rs.uniform(0.1, 3.0, size=shape[cdim])
        shp = [1] * len(shape)
        shp[cdim] = shape[cdim]
        x = x * sc.reshape(shp) + 0.25 * sc.reshape(shp)
    if relu:
        x = np.maximum(x, 0)
    return x.astype(np.float32)


def regen(spec):
    """Rebuild a fixture input from the ``input`` entry of ref_cpu_meta.json."""
    x = make_input(spec["seed"], tuple(spec["shape"]), spec.get("dist", "normal"), spec.get("relu", False),
                   spec.get("chan_scale", True))
    if "mult" in spec:
        x = (x * spec["mult"]).astype(np.float32)
    if "const_row" in spec:
        r, v = spec["const_row"]
        x[r, :] = v
    return x


# ---- the reference's compiled kernel (kernels/gemmlowp.cu), tests/test_gpu_ref_ext.py ------------------------------
F2G_SIZES = (1, 5, 1024, 100003, 1 << 22)
F2G_BITS = (2, 4, 8)
# (enforce_true_zero, range, offset) of every float2gemmlowp call per (n, bits), each without and with a noise tensor
F2G_CALLS = ((True, 7.3, -3.1), (False, 5.0, 0.0), (False, 6.0, 0.5), (True, 9.0, -1e-4), (False, 4.0, -1.0),
             (True, 1e-3, -4e-4), (True, 300.0, -150.0))


def f2g_inputs(n, bits):
    """(x, noise) float32 arrays of one float2gemmlowp case."""
    rs = np.random.RandomState(n + bits)
    x = (rs.standard_normal(n) * 2 + 0.3).astype(np.float32)
    noise = (rs.uniform(size=n) - 0.5).astype(np.float32)
    return x, noise


def f2g_key(n, bits, call, noise, int_exp=False):
    tz, rng, off = call
    return "n%d_b%d_tz%d_r%r_o%r_noise%d_ie%d" % (n, bits, tz, rng, off, noise, int_exp)


# gemmlowpMinMaxQuantize cases: (shape, tag, positive); input = standard normal (seed 5 + index), ReLU when positive
MINMAX_CASES = (((8, 16, 14, 14), "activation", False), ((8, 16, 14, 14), "activation", True),
                ((4, 1000), "activation_classifier", False), ((64, 32, 3, 3), "weight", False))


def minmax_input(i):
    shape, _, positive = MINMAX_CASES[i]
    x = np.random.RandomState(5 + i).standard_normal(shape).astype(np.float32)
    return np.maximum(x, 0) if positive else x
