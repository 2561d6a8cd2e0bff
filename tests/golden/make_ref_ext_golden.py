#!/usr/bin/env python
"""Record what the REFERENCE's own compiled kernel computes (kernels/gemmlowp.cu via int_quantization.float2gemmlowp) on
the inputs of tests/test_gpu_ref_ext.py, so that the test holds our kernels to the reference without needing the
reference's binary.  Needs a GPU and the extension oracle/build_oracle.py built for it:

    python tests/golden/make_ref_ext_golden.py      # writes tests/golden/ref_ext_float2gemmlowp.json, ref_ext_minmax.npz

float2gemmlowp outputs are stored as SHA-256 digests of their bytes (the test compares bit for bit); the min/max outputs as
their distinct float32 values plus one uint8 index per element (an 8-bit grid has at most 256 levels) and
the range the reference's host logic chose.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import golden_inputs as G  # noqa: E402
from oracle import ref_live  # noqa: E402


def digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    ext = ref_live.load_extension()
    out = {}
    for n in G.F2G_SIZES:
        for bits in G.F2G_BITS:
            xn, nn = G.f2g_inputs(n, bits)
            x, noise = torch.from_numpy(xn).cuda(), torch.from_numpy(nn).cuda()
            zeros = torch.zeros_like(x)
            for call in G.F2G_CALLS:
                tz, rng, off = call
                for nz in (zeros, noise):
                    out[G.f2g_key(n, bits, call, nz is noise)] = digest(ext.float2gemmlowp(x, rng, off, bits, False, tz, nz))
            call = (True, 7.3, -3.1)
            out[G.f2g_key(n, bits, call, False, int_exp=True)] = digest(ext.float2gemmlowp(x, 7.3, -3.1, bits, True, True, zeros))
    torch.cuda.synchronize()
    with open(os.path.join(HERE, "ref_ext_float2gemmlowp.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    # gemmlowpMinMaxQuantize (int_quantizer.py:361-379, 605-614): the reference's host logic, its kernel as the leaf
    arrays = {}
    for i, (shape, tag, positive) in enumerate(G.MINMAX_CASES):
        x = torch.from_numpy(G.minmax_input(i)).cuda()
        avg = "activation" in tag and "classifier" not in tag
        t = x.view(x.shape[0], -1) if avg else x.view(-1)
        mn = t.min(-1)[0].mean() if avg else t.min()
        mx = t.max(-1)[0].mean() if avg else t.max()
        if positive:
            mn = 0
        delta = mx - mn
        preserve_zero = bool((mn + delta) > 0 and mn < 0)
        want = ext.float2gemmlowp(x.contiguous(), float(delta), float(mn), 8, False, preserve_zero, torch.zeros_like(x))
        levels, codes = np.unique(want.cpu().numpy(), return_inverse=True)
        assert levels.size <= 256
        arrays["levels_%d" % i] = levels.astype(np.float32)
        arrays["codes_%d" % i] = codes.reshape(shape).astype(np.uint8)
        arrays["delta_%d" % i] = np.float64(float(delta))
    np.savez_compressed(os.path.join(HERE, "ref_ext_minmax.npz"), **arrays)


if __name__ == "__main__":
    main()
