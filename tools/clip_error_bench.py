#!/usr/bin/env python
"""The cost of the clipping-error columns (collect_err), timed on the GPU.  Writes one JSON object (--out) and prints it,
followed by the row profiles/README.md keeps for it.

  * ops.clip_error on a 512 x 64 x 112 x 112 tensor (the ResNet-50 stem output at batch 512) per tensor, per channel on
    NCHW memory and per channel on channels-last memory: CUDA events around each call after a warm-up, in GB/s
    (4 B/element, one read) and as a fraction of the H100 SXM data sheet's 3.35 TB/s;
  * one ResNet-50 `-sm collect` step (int4 activations) at batch 512, NCHW as the collect path runs, with and without
    collect_err, alternated round by round in the same process (each step ends in the statistics' host copies).
Writing the summary files (once per run) is not measured.
"""
import argparse
import json
import os
import tempfile
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_clip_error_bench.json"))
    a = ap.parse_args()
    build_or_exit("clip_error_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline

    # -- the kernel alone ------------------------------------------------------------------------------------------------
    n = a.batch
    x = torch.randn(n, 64, 112, 112, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    nbytes = 4.0 * x.numel()
    kernel = {}
    for name, t, layout, cl in (("per_tensor", x, (1, 1, x.numel()), False), ("per_channel_nchw", x, (n, 64, 112 * 112), False),
                                ("per_channel_channels_last", None, (n, 64, 112 * 112), True)):
        if t is None:
            t = x.contiguous(memory_format=torch.channels_last)
        table = ops.fused(t, layout, stats_only=True, channels_last=cl)
        for _ in range(3):
            ops.clip_error(t, table, layout, cl, 4, False)
        torch.cuda.synchronize()
        k = median(timed(lambda: ops.clip_error(t, table, layout, cl, 4, False), a.reps))
        kernel[name] = {"ms_median": round(k, 4), "gb_s": round(nbytes / (k * 1e-3) / 1e9, 1),
                        "hbm_fraction": round(nbytes / (k * 1e-3) / HBM_PEAK, 3)}
        del t, table
    del x
    torch.cuda.empty_cache()

    # -- one ResNet-50 collect step, with and without collect_err ---------------------------------------------------------------
    xb, _ = pipeline.synthetic_batch(n, seed=1, device="cuda")
    step = {False: [], True: []}
    with tempfile.TemporaryDirectory() as tmp:
        models = {}
        for err in (False, True):
            cfg = dict(arch="resnet50", qtype="int4", qweight="int4", stats_mode="collect", stats_folder="r50_%d" % err,
                       stats_base_dir=tmp, collect_err=err)
            models[err] = pipeline.build_quantized_model(cfg, "cuda")
        with torch.no_grad():
            for err in (False, True):
                models[err][0](xb)
            torch.cuda.synchronize()
            for _ in range(a.rounds):
                for err in (False, True):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    models[err][0](xb)
                    torch.cuda.synchronize()
                    step[err].append((time.perf_counter() - t0) * 1e3)
            ops.profile_reset(enable=True)
            models[True][0](xb)
            prof = ops.profile_collect()
            ops.profile_reset(enable=False)
        for err in (False, True):
            models[err][1].detach()
    e = prof["modes"].get("E", {"launches": 0, "ms": 0.0, "elems": 0})
    off, on = median(step[False]), median(step[True])
    res = {
        "tool": "clip_error_bench", "gpu": gpu_info(), "shape": [n, 64, 112, 112], "num_bits": 4,
        "clip_error": kernel,
        "resnet50_collect_int4": {"batch": n, "rounds": a.rounds, "step_ms_without": round(off, 1),
                                  "step_ms_with": round(on, 1), "step_ms_without_all": [round(v, 1) for v in step[False]],
                                  "step_ms_with_all": [round(v, 1) for v in step[True]],
                                  "clip_error_launches": e["launches"], "clip_error_ms": round(e["ms"], 2)},
        "note": "hbm fraction against the 3.35 TB/s data sheet, 4 B/element; collect steps are host-clock times around a "
                "synchronised forward (the collect path reads statistics back to the host per hooked tensor)",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    k, r = res["clip_error"], res["resnet50_collect_int4"]
    print("| `h100_clip_error_bench.json` | `python tools/clip_error_bench.py`: collect_err cost. Taken on %s. `ops.clip_error` "
          "on %dx64x112x112 (int4): per tensor %.0f GB/s (%.2f of 3.35 TB/s), per channel NCHW %.0f GB/s (%.2f), per channel "
          "channels-last %.0f GB/s (%.2f). ResNet-50 int4 collect at batch %d: %.0f ms per step without, %.0f ms with "
          "collect_err (%d clip_error launches, %.1f ms) |"
          % (res["gpu"], n, k["per_tensor"]["gb_s"], k["per_tensor"]["hbm_fraction"], k["per_channel_nchw"]["gb_s"],
             k["per_channel_nchw"]["hbm_fraction"], k["per_channel_channels_last"]["gb_s"],
             k["per_channel_channels_last"]["hbm_fraction"], n, off, on, r["clip_error_launches"], r["clip_error_ms"]))


if __name__ == "__main__":
    main()
