#!/usr/bin/env python
"""Activation norm fixtures (`-ms`) from the REAL reference (build container only).

The unmodified reference runs the seeded ResNet-18 of make_stats_golden.py (2 batches of 2 images, 64x64) with
`measure_stats` on, in four configurations.  Its distance_stats.MeasureStatistics writes <base>/distance/resnet18/
distance.csv on exit; `base_dir` is pointed at a scratch directory and each file is copied to
ref_distance/<config>/distance.csv.  The compiled leaf runs on the CPU restatement, as in make_census.py.
"""
import os
import shutil
import sys

import pandas as pd
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_stats_golden as msg  # noqa: E402  (reference import, stubs, CPU leaf, scratch statistics directory)

from pytorch_quantizer.quantization.inference import distance_stats as ds_mod  # noqa: E402

OUT = os.path.join(HERE, "ref_distance")
ds_mod.base_dir = msg.SCRATCH

CONFIGS = {
    "w4a4": dict(msg.W4A4),
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
    "collect": dict(stats_mode="collect", qtype="int4", qweight="int4"),
}


def main():
    torch.set_num_threads(8)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    shutil.rmtree(OUT, ignore_errors=True)
    xs = msg.batches()
    for name, flags in CONFIGS.items():
        msg.run(dict(measure_stats=True, **flags), xs)
        os.makedirs(os.path.join(OUT, name))
        src = os.path.join(msg.SCRATCH, "distance", "resnet18", "distance.csv")
        shutil.copy(src, os.path.join(OUT, name))
        df = pd.read_csv(src)
        print(name, df.shape, list(df.columns)[:4], "...")
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)


if __name__ == "__main__":
    main()
