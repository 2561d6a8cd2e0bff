#!/usr/bin/env python
"""The cost of the activation norm measurement (`-ms`), timed on the GPU.  Writes one JSON object (--out) and prints it,
followed by the row profiles/README.md keeps for it.

  * ops.sample_sumsq on a 512 x 64 x 112 x 112 tensor (the ResNet-50 stem output at batch 512): CUDA events around each
    call after a warm-up, in GB/s (4 B/element) and as a fraction of the H100 SXM data sheet's 3.35 TB/s;
  * the reference's per-tensor form, torch.sum(t**2, dim=-1).cpu() on t = x.view(N, -1), on the same tensor (it
    includes its device-to-host copy and the host synchronisation);
  * ResNet-50 W4A4 (BASELINE configs[2]) channels-last at batch 512, inputs resident: images/s with `-ms` off and on,
    alternated round by round in the same process, and the time the 'M' launches of one `-ms` forward take (the extra
    read pass); the rest of the difference is the three fusions `-ms` switches off.
Writing distance.csv (once per run) is not measured.
"""
import argparse
import json
import os
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5, help="forwards per config per round")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_measure_bench.json"))
    a = ap.parse_args()
    build_or_exit("measure_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True

    # -- the kernel alone ------------------------------------------------------------------------------------------------
    x = torch.randn(a.batch, 64, 112, 112, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    nbytes = 4.0 * x.numel()
    for _ in range(3):
        ops.sample_sumsq(x)
    torch.cuda.synchronize()
    k_ms = timed(lambda: ops.sample_sumsq(x), a.reps)
    t = x.view(x.shape[0], -1)
    for _ in range(3):
        torch.sum(t ** 2, dim=-1).cpu()
    ref_ms = []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch.sum(t ** 2, dim=-1).cpu()
        ref_ms.append((time.perf_counter() - t0) * 1e3)
    del x, t
    torch.cuda.empty_cache()

    # -- ResNet-50 W4A4 channels-last, -ms off / on ---------------------------------------------------------------------------
    cfg = pipeline.CONFIGS["resnet50_w4a4"]
    xb, _ = pipeline.synthetic_batch(a.batch, seed=1, device="cuda", channels_last=True)
    models = {}
    for ms in (False, True):
        models[ms] = pipeline.build_quantized_model(dict(cfg, measure_stats=ms), "cuda", channels_last=True)
    with torch.no_grad():
        for ms in (False, True):
            for _ in range(3):
                models[ms][0](xb)
        torch.cuda.synchronize()
        rates = {False: [], True: []}
        for _ in range(a.rounds):
            for ms in (False, True):
                model, qm = models[ms]
                ms_t = timed(lambda: [model(xb) for _ in range(a.steps)], 1)[0]
                rates[ms].append(a.batch * a.steps / (ms_t * 1e-3))
                if qm.measure_stats is not None:
                    qm.measure_stats.stats = {}   # keep only what one round measured
        ops.profile_reset(enable=True)
        models[True][0](xb)
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
    m = prof["modes"].get("M", {"launches": 0, "ms": 0.0, "elems": 0})
    off, on = median(rates[False]), median(rates[True])
    step_off, step_on = a.batch / off * 1e3, a.batch / on * 1e3
    res = {
        "tool": "measure_bench", "gpu": gpu_info(),
        "sample_sumsq": {"shape": [a.batch, 64, 112, 112], "ms_median": round(median(k_ms), 4),
                         "gb_s": round(nbytes / (median(k_ms) * 1e-3) / 1e9, 1),
                         "hbm_fraction": round(nbytes / (median(k_ms) * 1e-3) / HBM_PEAK, 3)},
        "reference_form": {"expr": "torch.sum(t**2, dim=-1).cpu()", "ms_median": round(median(ref_ms), 3),
                           "gb_s": round(nbytes / (median(ref_ms) * 1e-3) / 1e9, 1)},
        "resnet50_w4a4_cl": {"batch": a.batch, "rounds": a.rounds, "steps_per_round": a.steps,
                             "images_per_s_ms_off": round(off, 1), "images_per_s_ms_on": round(on, 1),
                             "images_per_s_off_all": [round(v, 1) for v in rates[False]],
                             "images_per_s_on_all": [round(v, 1) for v in rates[True]],
                             "step_ms_off": round(step_off, 2), "step_ms_on": round(step_on, 2),
                             "overhead_ms": round(step_on - step_off, 2),
                             "overhead_fraction": round(step_on / step_off - 1, 4),
                             "measure_launches": m["launches"], "measure_pass_ms": round(m["ms"], 2),
                             "measure_pass_gb_s": round(4.0 * m["elems"] / (m["ms"] * 1e-3) / 1e9, 1) if m["ms"] else None,
                             "fusions_off_ms_derived": round(step_on - step_off - m["ms"], 2)},
        "note": "hbm fraction against the 3.35 TB/s data sheet, 4 B/element; fusions_off_ms_derived = overhead minus the "
                "'M' launches' event time of one profiled forward (derived, not timed on its own); the distance.csv write "
                "is not measured",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    r = res["resnet50_w4a4_cl"]
    print("| `h100_measure_bench.json` | `python tools/measure_bench.py`: `-ms` cost. Taken on %s. `ops.sample_sumsq` on "
          "%dx64x112x112: %.1f GB/s (%.2f of 3.35 TB/s); the reference's `(t**2).sum(-1).cpu()`: %.1f GB/s. ResNet-50 W4A4 "
          "channels-last at batch %d: %.0f images/s without `-ms`, %.0f with it (+%.1f %% step time: %d measure launches "
          "%.2f ms, the three fusions switched off %.2f ms, derived) |"
          % (res["gpu"], a.batch, res["sample_sumsq"]["gb_s"], res["sample_sumsq"]["hbm_fraction"],
             res["reference_form"]["gb_s"], a.batch, off, on, 100 * r["overhead_fraction"], r["measure_launches"],
             r["measure_pass_ms"], r["fusions_off_ms_derived"]))


if __name__ == "__main__":
    main()
