#!/usr/bin/env python
"""The cost of k-means weight quantization (ops.kmeans1d, csrc/fq_kmeans.cuh), timed on the GPU.  Writes one JSON object
(--out) and prints it.

For every tensor kmeans_quantization.is_ignored lets through, of the seeded, BN-folded ResNet-50 at 4 and 8 bits and
VGG-16 at 4 bits (quantize task):
  * the whole launch (k-means++ and Lloyd): CUDA events around the library call (ops' profile mode 'C'), the median of
    --reps calls after one warm-up call on the same tensor; the host's k-means++ draws (ops.kmeans_draws, numpy) timed
    on their own with a host clock;
  * Lloyd alone: the same launch started from the k-means++ centres (init=), over n_iter gives the time per iteration;
    its effective read rate counts 4 B/element for every pass over the tensor (mean, variance, n_iter Lloyd passes,
    the last pass), against the H100 SXM data sheet's 3.35 TB/s;
  * scikit-learn 1.9's KMeans(n_clusters=k, random_state=0).fit on the host, beside it, for --sk tensors per
    configuration (the smallest ones; the reference script's own call).
The input check of ops.kmeans1d (one host synchronisation) and the draws are outside the events.
"""
import argparse
import json
import os
import time

import numpy as np

from benchlib import ROOT, build_or_exit, gpu_info, write_json

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def timed(fn, reps):
    """Median device time of the launch: the CUDA events ops.kmeans1d records around the library call (profile mode 'C'),
    so the host's input check and random draws stay outside."""
    from cnn_quantization_b200 import ops
    ms = []
    for _ in range(reps):
        ops.profile_reset(True)
        r = fn()
        ms.append(ops.profile_collect()["modes"]["C"]["ms"])
    ops.profile_reset(False)
    return float(np.median(ms)), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_kmeans_bench.json"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sk", type=int, default=3)
    ap.add_argument("--configs", default="resnet50:4,resnet50:8,vgg16:4")
    a = ap.parse_args()
    build_or_exit("kmeans_bench.py")
    import torch
    import cnn_quantization_b200 as fq
    from cnn_quantization_b200 import kmeans_quantization as KQ
    ops = fq.ops
    res = {"gpu": gpu_info(), "reps": a.reps, "configs": {}}
    for cfg in a.configs.split(","):
        arch, bits = cfg.split(":")
        bits = int(bits)
        model = KQ.build_model(arch, device="cpu")
        tensors = [(n, p.detach()) for n, p in model.named_parameters() if not KQ.is_ignored(n, p)]
        rows, tot = [], {"elements": 0, "ms_total": 0.0, "ms_lloyd": 0.0, "iters": 0, "host_draws_ms": 0.0}
        for name, w in tensors:
            x = w.cuda().contiguous()
            full = lambda: ops.kmeans1d(x, bits, task="quantize")   # noqa: E731
            full()
            torch.cuda.synchronize()
            ms, r = timed(full, a.reps)
            t0 = time.perf_counter()
            ops.kmeans_draws(x.numel(), 1 << bits, 0)
            host_ms = 1e3 * (time.perf_counter() - t0)
            init = x.reshape(-1)[r.init_ids].double()   # the k-means++ centres: the data values at the init indices
            lloyd = lambda: ops.kmeans1d(x, bits, task="quantize", init=init)   # noqa: E731
            lloyd()
            torch.cuda.synchronize()
            ms_l, rl = timed(lloyd, a.reps)
            it = int(rl.n_iter)
            n = x.numel()
            passes = it + 3
            row = {"name": name, "shape": list(w.shape), "n": n, "n_iter": int(r.n_iter), "ms": round(ms, 4), "host_draws_ms": round(host_ms, 3),
                   "ms_lloyd_from_init": round(ms_l, 4), "n_iter_from_init": it, "us_per_pass": round(1e3 * ms_l / passes, 3),
                   "read_GBps": round(4.0 * n * passes / (ms_l * 1e-3) / 1e9, 1),
                   "read_frac_peak": round(4.0 * n * passes / (ms_l * 1e-3) / HBM_PEAK, 3)}
            rows.append(row)
            tot["elements"] += n
            tot["ms_total"] += ms
            tot["host_draws_ms"] += host_ms
            tot["ms_lloyd"] += ms_l
            tot["iters"] += it
        try:
            from sklearn.cluster import KMeans
        except ImportError:   # the host comparison is optional
            KMeans = None
        order = sorted(range(len(tensors)), key=lambda i: tensors[i][1].numel())[:a.sk] if KMeans else []
        for i in order:
            xs = tensors[i][1].numpy().reshape(-1, 1)
            t0 = time.perf_counter()
            km = KMeans(n_clusters=1 << bits, random_state=0).fit(xs)
            rows[i]["sklearn_host_s"] = round(time.perf_counter() - t0, 3)
            rows[i]["sklearn_n_iter"] = int(km.n_iter_)
        res["configs"][cfg] = {"tensors": rows, "total": {k: (round(v, 3) if isinstance(v, float) else v) for k, v in tot.items()}}
        print(cfg, json.dumps(res["configs"][cfg]["total"]), flush=True)
        del model
    write_json(res, a.out)
    print(json.dumps(res)[:2000])


if __name__ == "__main__":
    main()
