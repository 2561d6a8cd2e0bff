"""Stand-alone kernel timing on the ResNet-50 activation census (not the bench contract; a development tool).

    python tools/microbench.py [--n 512] [--reps 5]
"""
import argparse
import sys

import torch

sys.path.insert(0, ".")
import cnn_quantization_b200 as fq  # noqa: E402
from cnn_quantization_b200 import _lib as L  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=512)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--shapes", default="all")
args = ap.parse_args()

N = args.n
census = [(64, 112), (64, 56), (256, 56), (128, 56), (128, 28), (512, 28), (256, 28), (256, 14), (1024, 14), (512, 14),
          (512, 7), (2048, 7)]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
PEAK = 3350.0  # H100 SXM data sheet, GB/s


def timeit(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


print("shape, mode, ms, Gelem/s, algorithmic GB/s, frac of %.0f" % PEAK)
for c, hw in census:
    x = torch.randn(N, c, hw, hw, device="cuda")
    out = torch.empty_like(x)
    n_el = x.numel()
    lay = (N, c, hw * hw)
    modes = [
        ("D laplace+ba (16B)", 16, lambda: fq.ops.fused(x, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, out=out)),
        ("D laplace+ba halfrange", 16, lambda: fq.ops.fused(x, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, positive=True, out=out)),
        ("B minmax pc torch-leaf (12B)", 12, lambda: fq.ops.fused(x, lay, range_mode=L.RANGE_MINMAX, num_bits=4, out=out)),
        ("B minmax per-sample compiled (12B)", 12, lambda: fq.ops.fused(x, (1, N, c * hw * hw), scope=L.SCOPE_GROUP_MEAN, leaf=L.LEAF_COMPILED, num_bits=8, out=out)),
    ]
    d = torch.rand(c, device="cuda") + 1
    o = -torch.rand(c, device="cuda")
    modes.append(("A given params (8B)", 8, lambda: fq.ops.quantize1(x, d, o, 4, layout=lay)))
    modes.append(("a1 float2gemmlowp (8B)", 8, lambda: fq.ops.float2gemmlowp(x, 7.0, -3.0, 8, False, True, None, out=out)))
    modes.append(("copy_ (8B)", 8, lambda: out.copy_(x)))
    for name, bpe, fn in modes:
        ms = timeit(fn, args.reps)
        gbs = n_el * bpe / ms / 1e6
        print("%dx%dx%dx%d, %s, %.3f, %.2f, %.0f, %.3f" % (N, c, hw, hw, name, ms, n_el / ms / 1e6, gbs, gbs / PEAK))
    del x, out
