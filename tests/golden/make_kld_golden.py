#!/usr/bin/env python
"""KL-divergence calibration fixtures from the REAL reference (build container only):

  1. ref_kld.npz: for every row of kld_oracle.fixture_rows() (kind, shape, seed), the reference's
     kld_threshold._get_optimal_threshold: its histogram, its full divergence curve, its index and its threshold;
  2. `-kld -sm collect` on the seeded ResNet-18 of make_stats_golden.py (2 batches of 2 images, 64x64, int4) -> the
     reference's summary CSV, copied to ref_stats_kld/statistics/resnet18_kld_int4/;
  3. `-kld -sm use` with those statistics -> logits in ref_stats_kld_logits.npz.

numpy >= 2 computes np.histogram's edges in float32 for float32 data (NEP 50), and the reference then fails its own
edge-symmetry assert.  The authors ran numpy 1.x, where the edges are the float64 linspace rounded to float32.  That is
the behaviour these fixtures record: in this process only, the `np` the reference's kld_threshold module sees is a
namespace whose histogram(a, bins, range) widens a degenerate range as numpy does, builds the numpy 1.x edges and
bins against them.  The same namespace records the divergence array the reference hands to np.argmin.  The reference's
code itself runs unmodified.
"""
import os
import shutil
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import kld_oracle as KO  # noqa: E402
import make_stats_golden as msg  # noqa: E402  (reference import, stubs, CPU leaf, scratch statistics directory)

from pytorch_quantizer.quantization.inference import kld_threshold as kt  # noqa: E402

OUT = os.path.join(HERE, "ref_stats_kld")
curves = []


def _histogram(a, bins, range):
    lo, hi = float(range[0]), float(range[1])
    if lo == hi:
        lo, hi = lo - 0.5, hi + 0.5
    edges = np.linspace(lo, hi, bins + 1).astype(np.float32)
    return np.histogram(a, bins=edges)


def _argmin(a, *args, **kw):
    curves.append(np.array(a, copy=True))
    return np.argmin(a, *args, **kw)


shim = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
shim.histogram = _histogram
shim.argmin = _argmin
kt.np = shim


def rows_fixture():
    rec = {k: [] for k in ("kind", "shape", "seed", "hist", "div", "idx", "th")}
    for kind, shape, seed in KO.fixture_rows():
        x = KO.make_row(kind, shape, seed)
        del curves[:]
        _, _, _, th = kt._get_optimal_threshold(x, num_bins=2001, num_quantized_bins=15)
        div = curves[-1]
        hist = _histogram(x, 2001, (-max(abs(x.min()), abs(x.max())), max(abs(x.min()), abs(x.max()))))[0]
        rec["kind"].append(kind)
        rec["shape"].append(list(shape))
        rec["seed"].append(seed)
        rec["hist"].append(hist.astype(np.int32))
        rec["div"].append(div.astype(np.float64))
        rec["idx"].append(int(np.argmin(div)))
        rec["th"].append(np.float32(th))
        print("%-8s %-14s idx %4d th %.6g div %.6g" % (kind, shape, rec["idx"][-1], th, div[rec["idx"][-1]]))
    np.savez_compressed(os.path.join(HERE, "ref_kld.npz"), kind=np.array(rec["kind"]), shape=np.array(rec["shape"]),
                        seed=np.array(rec["seed"]), hist=np.stack(rec["hist"]), div=np.stack(rec["div"]),
                        idx=np.array(rec["idx"], dtype=np.int32), th=np.array(rec["th"], dtype=np.float32))


KLD = dict(qtype="int4", qweight="int8", kld_threshold=True)


def main():
    torch.set_num_threads(8)
    rows_fixture()
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    xs = msg.batches()
    msg.run(dict(stats_mode="collect", **KLD), xs)
    logits = {"use_kld_int4": msg.run(dict(stats_mode="use", **KLD), xs)}
    shutil.rmtree(OUT, ignore_errors=True)
    folder = os.path.join(OUT, "statistics", "resnet18_kld_int4")
    os.makedirs(folder)
    shutil.copy(os.path.join(msg.SCRATCH, "statistics", "resnet18_kld_int4", "resnet18_kld_int4_summary.csv"), folder)
    np.savez_compressed(os.path.join(HERE, "ref_stats_kld_logits.npz"), **logits)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    for k, v in logits.items():
        print(k, v.shape, float(np.abs(v).mean()))


if __name__ == "__main__":
    main()
