#!/usr/bin/env python
"""The cost of measured weight clipping (`clip_weight="mse"`), timed on the GPU.  Writes one JSON object (--out) and
prints it.

  * quantize_model wall time (host clock around a synchronised call, after one warm-up call) on ResNet-50 and VGG-16 at
    `-qw int4 -pcq_w -bcw` with seeded random weights: the default min/max weights, `-baw -bap mse` alone (min/max at the
    widths bit_alloc.allocate gives on the host), clip_weight="mse", and clip_weight="mse" with `-baw -bap mse`;
  * ops.allocate_widths (CUDA events over 20 launches) against bit_alloc.allocate (host clock) on a random [2048, 9]
    table at target 4, and whether the widths are equal;
  * the candidate launches of one VGG-16 fc6 weight (4096 x 25088) at 4 bits: ops.clip_mse_grid over the 125 default
    multipliers at one width and at widths 0..8, and the min/max ops.clip_mse over widths 0..8 (CUDA events).
"""
import argparse
import copy
import json
import os
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_weight_mse_bench.json"))
    a = ap.parse_args()
    build_or_exit("weight_mse_bench.py")
    import numpy as np
    import torch
    import torchvision.models as models
    import cnn_quantization_b200.manager as M
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS

    configs = {"minmax": dict(), "baw_bap_mse": dict(bit_alloc_weight=True, bit_alloc_prior="mse"),
               "clip_mse": dict(clip_weight="mse"),
               "clip_mse_baw_bap_mse": dict(clip_weight="mse", bit_alloc_weight=True, bit_alloc_prior="mse")}
    qm_s = {}
    for arch in ("resnet50", "vgg16"):
        torch.manual_seed(12345)
        base = models.__dict__[arch](weights=None).eval().cuda()
        qm_s[arch] = {}
        for name, flags in configs.items():
            args = M.make_args(arch=arch, qtype="int4", qweight="int4", per_channel_quant_weights=True,
                               bias_corr_weight=True, **flags)
            ts = []
            for _ in range(1 + a.reps):
                qm = M.QuantizationManagerInference(args, M.get_params(args))
                model = copy.deepcopy(base)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                qm.quantize_model(model)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            qm_s[arch][name] = {"s_median": round(median(ts[1:]), 3), "s_all": [round(t, 3) for t in ts[1:]],
                                "s_first": round(ts[0], 3)}
        del base

    rs = np.random.RandomState(0)
    t = rs.exponential(size=(2048, 9)).cumsum(1)[:, ::-1].copy()
    td = torch.from_numpy(t).cuda()
    ops.allocate_widths(td, 4)
    dev_ms = median(timed(lambda: ops.allocate_widths(td, 4), 20))
    host = []
    for _ in range(3):
        t0 = time.perf_counter()
        want = allocate(t, 4)
        host.append(time.perf_counter() - t0)
    same = bool(np.array_equal(ops.allocate_widths(td, 4).cpu().numpy(), want.astype(np.float32)))

    w = torch.randn(4096, 25088, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 0.01
    layout = (1, 4096, 25088)
    table = ops.fused(w, layout, num_bits=4, stats_only=True)
    mult = torch.tensor(MSE_MULTIPLIERS, dtype=torch.float32).cuda()
    zeros = torch.zeros(9, device="cuda")
    launches = {
        "clip_mse_grid_1x125": lambda: ops.clip_mse_grid(w, table, layout, False, 4, False, mult, [4], want_params=True),
        "clip_mse_grid_9x125": lambda: ops.clip_mse_grid(w, table, layout, False, 4, False, mult, list(range(9)),
                                                         want_params=True),
        "clip_mse_minmax_9": lambda: ops.clip_mse(w, table, layout, False, 4, False, zeros, prior="minmax",
                                                  widths=list(range(9)), want_params=True),
    }
    fc6 = {}
    for name, fn in launches.items():
        fn()
        fc6[name + "_ms"] = round(median(timed(fn, 3)), 2)

    res = {
        "tool": "weight_mse_bench", "gpu": gpu_info(),
        "quantize_model_int4_pcq_w_bcw": qm_s,
        "allocate_widths_G2048_target4": {"device_ms_median": round(dev_ms, 3), "host_s_median": round(median(host), 3),
                                          "widths_equal": same},
        "vgg16_fc6_4096x25088_candidate_launches": fc6,
        "multipliers": len(MSE_MULTIPLIERS),
        "note": "quantize_model: host clock around a synchronised call after one warm-up call, seeded random weights; "
                "kernel times: CUDA events (median)",
    }
    write_json(res, a.out)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
