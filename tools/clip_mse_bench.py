#!/usr/bin/env python
"""The cost of the clipping-MSE curves (collect_mse), timed on the GPU.  Writes one JSON object (--out) and prints it,
followed by the row profiles/README.md keeps for it.

  * ops.clip_mse over the default 125 multipliers on a 512 x 64 x 112 x 112 tensor (the ResNet-50 stem output at batch
    512, the largest tensor of the network) per channel on channels-last memory and per tensor: CUDA events around each
    call after a warm-up, in candidate evaluations per second (elements x K), against the two bounds of the kernel - one
    float64 FMA per candidate and element at the H100 SXM data sheet's 34 TFLOP/s FP64 (17e12 FMA/s), and one read of
    the tensor at its 3.35 TB/s - naming the larger (the one that applies);
  * one ResNet-50 W4A4 `-sm collect` step on channels-last memory at batch 512, with and without collect_mse,
    alternated round by round in the same process (host clock around a synchronised forward), and the GPU time of all
    clip_mse launches of one step (CUDA events, ops profile mode 'R').
Writing the curve files (once per run) is not measured.
"""
import argparse
import json
import os
import tempfile
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json

HBM_PEAK = 3.35e12        # H100 SXM data sheet, bytes/s
FP64_FMA_PEAK = 34e12 / 2  # H100 SXM data sheet FP64 (non-tensor) 34 TFLOP/s = 17e12 FMA/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_clip_mse_bench.json"))
    a = ap.parse_args()
    build_or_exit("clip_mse_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS

    # -- the kernel alone ------------------------------------------------------------------------------------------------
    n = a.batch
    mult = torch.tensor(MSE_MULTIPLIERS, dtype=torch.float32, device="cuda")
    k = mult.numel()
    x = torch.randn(n, 64, 112, 112, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    x = x.contiguous(memory_format=torch.channels_last)
    evals = float(x.numel()) * k
    t_fma, t_hbm = evals / FP64_FMA_PEAK, 4.0 * x.numel() / HBM_PEAK
    kernel = {}
    for name, layout, cl in (("per_channel_channels_last", (n, 64, 112 * 112), True), ("per_tensor", (1, 1, x.numel()), False)):
        table = ops.fused(x, layout, stats_only=True, channels_last=cl, any_dense_format=not cl)
        ops.clip_mse(x, table, layout, cl, 4, True, mult)
        torch.cuda.synchronize()
        ms = median(timed(lambda: ops.clip_mse(x, table, layout, cl, 4, True, mult), a.reps))
        rate = evals / (ms * 1e-3)
        kernel[name] = {"ms_median": round(ms, 2), "candidate_evals_per_s": float("%.4g" % rate),
                        "fraction_of_fp64_fma_bound": round(t_fma / (ms * 1e-3), 3),
                        "fraction_of_hbm_bound": round(t_hbm / (ms * 1e-3), 4)}
        del table
    del x
    torch.cuda.empty_cache()

    # -- one ResNet-50 W4A4 collect step on channels-last memory, with and without collect_mse ---------------------------------------
    xb, _ = pipeline.synthetic_batch(n, seed=1, device="cuda", channels_last=True)
    step = {False: [], True: []}
    with tempfile.TemporaryDirectory() as tmp:
        models = {}
        for on in (False, True):
            cfg = dict(pipeline.CONFIGS["resnet50_w4a4"], stats_mode="collect", stats_folder="r50_%d" % on,
                       stats_base_dir=tmp, collect_mse=on)
            models[on] = pipeline.build_quantized_model(cfg, "cuda", channels_last=True)
        with torch.no_grad():
            for on in (False, True):
                models[on][0](xb)
            torch.cuda.synchronize()
            for _ in range(a.rounds):
                for on in (False, True):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    models[on][0](xb)
                    torch.cuda.synchronize()
                    step[on].append(time.perf_counter() - t0)
            ops.profile_reset(enable=True)
            models[True][0](xb)
            prof = ops.profile_collect()
            ops.profile_reset(enable=False)
        for on in (False, True):
            models[on][1].detach()
    r = prof["modes"].get("R", {"launches": 0, "ms": 0.0, "elems": 0})
    off, on = median(step[False]), median(step[True])
    res = {
        "tool": "clip_mse_bench", "gpu": gpu_info(), "shape": [n, 64, 112, 112], "num_bits": 4, "multipliers": k,
        "bounds": {"fp64_fma_ms": round(t_fma * 1e3, 2), "hbm_read_ms": round(t_hbm * 1e3, 3),
                   "applies": "fp64_fma" if t_fma > t_hbm else "hbm"},
        "clip_mse": kernel,
        "resnet50_w4a4_collect_channels_last": {
            "batch": n, "rounds": a.rounds, "s_per_batch_without": round(off, 3), "s_per_batch_with": round(on, 3),
            "s_per_batch_without_all": [round(v, 3) for v in step[False]],
            "s_per_batch_with_all": [round(v, 3) for v in step[True]],
            "clip_mse_launches": r["launches"], "clip_mse_gpu_ms": round(r["ms"], 1),
            "clip_mse_candidate_evals": float("%.4g" % (float(r["elems"]) * k))},
        "note": "candidate evaluations = elements x multipliers; bounds from the H100 SXM data sheet (34 TFLOP/s FP64 = one "
                "FMA per evaluation at 17e12/s; 3.35 TB/s for one 4 B/element read), not measured; collect steps are "
                "host-clock times around a synchronised forward",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    kc, kt, c = res["clip_mse"]["per_channel_channels_last"], res["clip_mse"]["per_tensor"], res["resnet50_w4a4_collect_channels_last"]
    print("| `h100_clip_mse_bench.json` | `python tools/clip_mse_bench.py`: collect_mse cost. Taken on %s. `ops.clip_mse` "
          "(K = %d) on %dx64x112x112 channels-last (int4, positive): per channel %.3g candidate evaluations/s (%.2f of the "
          "FP64 FMA bound, which applies; %.4f of the one-read HBM bound), per tensor %.3g/s (%.2f). ResNet-50 W4A4 collect "
          "at batch %d, channels-last: %.2f s per batch without, %.2f s with collect_mse (%d clip_mse launches, %.0f ms GPU) |"
          % (res["gpu"], k, n, kc["candidate_evals_per_s"], kc["fraction_of_fp64_fma_bound"], kc["fraction_of_hbm_bound"],
             kt["candidate_evals_per_s"], kt["fraction_of_fp64_fma_bound"], n, off, on, c["clip_mse_launches"],
             c["clip_mse_gpu_ms"]))


if __name__ == "__main__":
    main()
