#!/usr/bin/env python
"""Sample-angle fixtures (`-ms` with the reference's angle_stats module) from the REAL reference (build container only).

The unmodified reference runs the seeded ResNet-18 of make_stats_golden.py with `measure_stats` on, in four
configurations, with its manager's `MS` rebound to angle_stats.MeasureStatistics - the reference's own way of selecting
the angle measurement (the commented import at inference_quantization_manager.py:10-11).  Its own seeded batches: 2 batches
of 6 images, 64x64, so every matrix holds 15 pairs per batch.  angle_stats writes <base>/angle/resnet18/angle.pkl on exit
({id: DataFrame, ..., 'target': []}); `base_dir` is pointed at a scratch directory and each pickle is converted to
ref_angle/<config>.npz (one float64 array per id, `ids` in the pickle's order, `target`), which keeps pickled pandas
objects out of the tree.  The compiled leaf runs on the CPU restatement, as in make_census.py.
"""
import os
import pickle
import shutil
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_stats_golden as msg  # noqa: E402  (reference import, stubs, CPU leaf, scratch statistics directory)

from pytorch_quantizer.quantization.inference import angle_stats as as_mod  # noqa: E402

OUT = os.path.join(HERE, "ref_angle")
as_mod.base_dir = msg.SCRATCH
msg.mc.iqm.MS = as_mod.MeasureStatistics

CONFIGS = {
    "w4a4": dict(msg.W4A4),
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
    "collect": dict(stats_mode="collect", qtype="int4", qweight="int4"),
}


def batches():
    rs = np.random.RandomState(2025)
    return [torch.from_numpy(rs.standard_normal((6, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def main():
    torch.set_num_threads(8)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    xs = batches()
    for name, flags in CONFIGS.items():
        msg.run(dict(measure_stats=True, **flags), xs)
        with open(os.path.join(msg.SCRATCH, "angle", "resnet18", "angle.pkl"), "rb") as f:
            d = pickle.load(f)
        ids = [k for k in d if k != "target"]
        arrays = {"id%03d" % i: d[k].to_numpy(dtype=np.float64) for i, k in enumerate(ids)}
        np.savez_compressed(os.path.join(OUT, name + ".npz"), ids=np.array(ids),
                            target=np.asarray(d["target"], dtype=np.float64), **arrays)
        print(name, len(ids), arrays["id000"].shape, ids[:3], "...")
        shutil.rmtree(os.path.join(msg.SCRATCH, "angle"), ignore_errors=True)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)


if __name__ == "__main__":
    main()
