#!/usr/bin/env python
"""The cost of the quantization-noise measurement (`-ms` with measure_stats_kind="noise"), timed on the GPU.  Writes one
JSON object (--out) and prints it, followed by the row profiles/README.md keeps for it.

  * ops.sample_noise stand-alone, with q: 512x64x112x112 channels-last with a convolution bias (the ResNet-50 stem's
    output) and 512x2048x7x7 (its last block): CUDA-event time per call, the bytes it must read (8 B/element) over that
    time, and that rate against the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth, which bounds this work (about 8
    float64 operations per element pair are far below the FP64 rate);
  * ResNet-50 W4A4 (BASELINE configs[2]) channels-last at batch 512, inputs resident: images/s with measurement off, with
    the norm kind and with the noise kind, alternated round by round in one process, with the logits checked equal;
  * the CUDA-event time of the 'N' launches of one profiled noise forward.
Writing the CSV files (once per run) is not measured.
"""
import argparse
import json
import os

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json

HBM_PEAK = 3.35e12   # H100 SXM data sheet, HBM3, B/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2, help="forwards per arm per round")
    ap.add_argument("--reps", type=int, default=20, help="timed stand-alone calls per shape")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_noise_bench.json"))
    a = ap.parse_args()
    build_or_exit("noise_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gpu = gpu_info()

    standalone = {}
    g = torch.Generator(device="cuda").manual_seed(5)
    for name, shape, cl, with_bias in (("stem_64x112x112_cl_bias", (a.batch, 64, 112, 112), True, True),
                                       ("last_2048x7x7", (a.batch, 2048, 7, 7), False, False)):
        y = torch.randn(shape, device="cuda", generator=g)
        if cl:
            y = y.contiguous(memory_format=torch.channels_last)
        q = torch.round(y * 4) / 4
        bias = torch.randn(shape[1], device="cuda", generator=g) if with_bias else None
        period = (-shape[1] if cl else shape[2] * shape[3]) if with_bias else 0
        call = lambda: ops.sample_noise(y, q, bias, period)
        for _ in range(3):
            call()
        ms = median(timed(call, a.reps))
        nbytes = 8 * y.numel()
        standalone[name] = {"shape": list(shape), "channels_last": cl, "bias": with_bias, "ms": round(ms, 3),
                            "gb_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                            "fraction_of_3_35_tb_s": round(nbytes / (ms * 1e-3) / HBM_PEAK, 3)}
        del y, q

    cfg = pipeline.CONFIGS["resnet50_w4a4"]
    xb, _ = pipeline.synthetic_batch(a.batch, seed=1, device="cuda", channels_last=True)
    arms = {"off": dict(cfg), "distance": dict(cfg, measure_stats=True),
            "noise": dict(cfg, measure_stats=True, measure_stats_kind="noise")}
    models = {k: pipeline.build_quantized_model(v, "cuda", channels_last=True) for k, v in arms.items()}

    def forget(qm):   # keep only what one round measured
        if qm.measure_stats is not None:
            qm.measure_stats.stats = {}

    logits = {}
    with torch.no_grad():
        for k, (model, qm) in models.items():
            logits[k] = model(xb).clone()
            forget(qm)
        torch.cuda.synchronize()
        rates = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, (model, qm) in models.items():
                t = timed(lambda: [model(xb) for _ in range(a.steps)])[0]
                rates[k].append(a.batch * a.steps / (t * 1e-3))
                forget(qm)
        ops.profile_reset(enable=True)
        models["noise"][0](xb)
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        forget(models["noise"][1])
    equal = all(torch.equal(logits["off"], logits[k]) for k in ("distance", "noise"))
    n = prof["modes"].get("N", {"launches": 0, "ms": 0.0, "bytes": 0})
    res = {
        "tool": "noise_bench", "gpu": gpu, "batch": a.batch,
        "sample_noise_standalone": standalone,
        "resnet50_w4a4_cl": {"rounds": a.rounds, "steps_per_round": a.steps,
                             "images_per_s": {k: round(median(v), 1) for k, v in rates.items()},
                             "images_per_s_all": {k: [round(x, 1) for x in v] for k, v in rates.items()},
                             "logits_equal_across_arms": equal,
                             "noise_launches_per_forward": n["launches"], "noise_ms_per_forward": round(n["ms"], 2),
                             "noise_gb_s": round(n["bytes"] / (n["ms"] * 1e-3) / 1e9, 1) if n["ms"] else None},
        "note": "stand-alone: median CUDA-event time of one call with q, bytes = 8 per element (y and q read once); "
                "per forward: the 'N' launches (output with its quantized form, input, each weight once per model) of "
                "one profiled forward; the data-sheet 3.35 TB/s is the bound, not a figure reached",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    s, r = standalone, res["resnet50_w4a4_cl"]
    print("| `h100_noise_bench.json` | `python tools/noise_bench.py`: the noise kind of `-ms`. Taken on %s. `sample_noise` "
          "stand-alone at batch %d: %.0f GB/s (%.2f of 3.35 TB/s) on 64x112x112 channels-last with bias, %.0f GB/s "
          "(%.2f) on 2048x7x7. ResNet-50 W4A4 channels-last: %d `N` launches %.1f ms per forward; %.0f images/s off, "
          "%.0f with the norm kind, %.0f with the noise kind |"
          % (gpu, a.batch, s["stem_64x112x112_cl_bias"]["gb_s"], s["stem_64x112x112_cl_bias"]["fraction_of_3_35_tb_s"],
             s["last_2048x7x7"]["gb_s"], s["last_2048x7x7"]["fraction_of_3_35_tb_s"], r["noise_launches_per_forward"],
             r["noise_ms_per_forward"], r["images_per_s"]["off"], r["images_per_s"]["distance"],
             r["images_per_s"]["noise"]))
    if not equal:
        raise SystemExit("logits differ across the arms")


if __name__ == "__main__":
    main()
