#!/usr/bin/env python
"""The cost of `-c mse` on the fly (`-sm no`), timed on the GPU.  Writes one JSON object (--out) and prints it, followed
by the row profiles/README.md keeps for it.

  * ResNet-50 W4A4 (`-pcq_w -pcq_a -baa -baw -bcw`) on channels-last memory at batch 512, in images per second, with
    `-c mse` over the default 125 multipliers and over 33 (2.0 .. 10.0 in steps of 0.25), alternated round by round in
    the same process with `-c laplace` on the same flags (host clock around a synchronised forward);
  * the GPU time of one forward of each, per launch mode of the ops launch profile (CUDA events; 'R' is the candidate
    sums with the selection, 'S' the statistics-only launches, 'A' the given-parameter applies);
  * the 512 x 64 x 112 x 112 stem tensor alone: ops.clip_mse_select against ops.clip_mse at both multiplier counts, the
    cost of the selection (CUDA events around each call after a warm-up).
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fly_mse_bench.json"))
    a = ap.parse_args()
    build_or_exit("fly_mse_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS

    n = a.batch
    short = [2.0 + 0.25 * i for i in range(33)]
    runs = {"laplace": dict(clipping="laplace"), "mse_k125": dict(clipping="mse"),
            "mse_k33": dict(clipping="mse", mse_multipliers=short)}

    # -- the stem tensor alone ------------------------------------------------------------------------------------------
    x = torch.randn(n, 64, 112, 112, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0)).relu_()
    x = x.contiguous(memory_format=torch.channels_last)
    layout = (n, 64, 112 * 112)
    table = ops.fused(x, layout, stats_only=True, channels_last=True, num_bits=4, positive=True, bit_alloc=True,
                      bit_alloc_target=4)
    stem = {}
    for name, m in (("k125", MSE_MULTIPLIERS), ("k33", short)):
        mult = torch.tensor(m, dtype=torch.float32, device="cuda")
        calls = {"clip_mse": lambda: ops.clip_mse(x, table, layout, True, 4, True, mult, bit_alloc=True),
                 "clip_mse_select": lambda: ops.clip_mse_select(x, table, layout, True, 4, True, mult, bit_alloc=True)}
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in calls}
        for _ in range(a.reps):   # alternated, so both see the same clocks
            for k, fn in calls.items():
                ms[k] += timed(fn)
        stem[name] = {k: round(median(v), 3) for k, v in ms.items()}
        stem[name]["selection_ms"] = round(stem[name]["clip_mse_select"] - stem[name]["clip_mse"], 3)
    del x, table
    torch.cuda.empty_cache()

    # -- ResNet-50 W4A4, channels-last, batch 512 ----------------------------------------------------------------------
    xb, _ = pipeline.synthetic_batch(n, seed=1, device="cuda", channels_last=True)
    models = {k: pipeline.build_quantized_model(dict(pipeline.CONFIGS["resnet50_w4a4"], **v), "cuda", channels_last=True)
              for k, v in runs.items()}
    step = {k: [] for k in runs}
    modes = {}
    with torch.no_grad():
        for k in runs:
            models[k][0](xb)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k in runs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                models[k][0](xb)
                torch.cuda.synchronize()
                step[k].append(time.perf_counter() - t0)
        for k in runs:
            ops.profile_reset(enable=True)
            models[k][0](xb)
            prof = ops.profile_collect()
            ops.profile_reset(enable=False)
            modes[k] = {m: {"launches": v["launches"], "gpu_ms": round(v["ms"], 2)} for m, v in sorted(prof["modes"].items())}
    for k in runs:
        models[k][1].detach()
    net = {k: {"images_per_s": round(n / median(step[k]), 1), "s_per_batch_all": [round(v, 4) for v in step[k]],
               "gpu_ms_per_mode": modes[k]} for k in runs}
    res = {
        "tool": "fly_mse_bench", "gpu": gpu_info(), "batch": n, "flags": "-pcq_w -pcq_a -baa -baw -bcw, int4, channels-last",
        "multipliers_k33": [short[0], short[-1], 0.25],
        "resnet50_w4a4": net,
        "stem_512x64x112x112_channels_last": stem,
        "note": "images/s from host-clock times around a synchronised forward, the three configurations alternated round "
                "by round; GPU times per launch mode from CUDA events in a separate profiled forward; stem times are "
                "CUDA-event medians, clip_mse_select and clip_mse alternated",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    r = res["resnet50_w4a4"]
    print("| `h100_fly_mse_bench.json` | `python tools/fly_mse_bench.py`: `-c mse` on the fly. Taken on %s. ResNet-50 W4A4 "
          "(`-baa -baw -bcw`) at batch %d, channels-last: %.0f images/s with `-c laplace`, %.0f with `-c mse` at 125 "
          "multipliers, %.0f at 33. Stem tensor alone at K = 125: clip_mse %.1f ms, clip_mse_select %.1f ms |"
          % (res["gpu"], n, r["laplace"]["images_per_s"], r["mse_k125"]["images_per_s"], r["mse_k33"]["images_per_s"],
             stem["k125"]["clip_mse"], stem["k125"]["clip_mse_select"]))


if __name__ == "__main__":
    main()
