#!/usr/bin/env python
"""The cost of the joint width-and-clip search (`-c mse -bap mse`), timed on the GPU.  Writes one JSON object (--out)
and prints it, followed by the row profiles/README.md keeps for it.

  * ops.clip_mse_grid over widths 0..8 x the 125 default multipliers (Laplace prior, positive) per channel on a
    512 x 64 x 112 x 112 channels-last tensor (the ResNet-50 stem output at batch 512): CUDA events around each call after
    a warm-up, against the five ops.clip_mse(widths=...) launches of at most 256 candidates over the same 1125 pairs, and
    whether the columns are equal;
  * one ResNet-50 W4A4 `-sm collect` step under `-c mse` on channels-last memory at batch 512, with collect_mse alone and
    with collect_mse + collect_bits, alternated round by round in the same process (host clock around a synchronised
    forward);
  * ResNet-50 W4A4 `-sm use` images/s on the collected batch: `-c mse -baa` (analytic widths) against `-c mse -baa -bap
    mse`, alternated in the same process (CUDA events around each forward).
Writing the statistics files (once per collect) is not measured.
"""
import argparse
import json
import os
import tempfile
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_joint_mse_bench.json"))
    a = ap.parse_args()
    build_or_exit("joint_mse_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS

    # -- the kernel alone ------------------------------------------------------------------------------------------------
    n = a.batch
    x = torch.randn(n, 64, 112, 112, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    x = torch.relu(x).contiguous(memory_format=torch.channels_last)
    layout = (n, 64, 112 * 112)
    table = ops.fused(x, layout, stats_only=True, channels_last=True)
    mult = torch.tensor(MSE_MULTIPLIERS, dtype=torch.float32, device="cuda")
    widths = list(range(9))
    pairs = [(w, k) for w in widths for k in range(mult.numel())]
    parts = [pairs[i:i + 256] for i in range(0, len(pairs), 256)]
    parts = [(mult[torch.tensor([k for _, k in p], device="cuda")], [w for w, _ in p]) for p in parts]
    grid = lambda: ops.clip_mse_grid(x, table, layout, True, 4, True, mult, widths, solve_f64=False)
    split = lambda: [ops.clip_mse(x, table, layout, True, 4, True, m, widths=w, solve_f64=False) for m, w in parts]
    grid(), split()
    torch.cuda.synchronize()
    ms_grid = median(timed(grid, a.reps))
    ms_split = median(timed(split, a.reps))
    g, s = grid(), split()
    same = torch.equal(g, torch.cat([s[0][:, :1]] + [p[:, 1:] for p in s], 1))
    evals = x.numel() * len(pairs)
    del g, s, x, table
    torch.cuda.empty_cache()

    # -- ResNet-50 W4A4 collect under -c mse: collect_mse alone, and with collect_bits; then use mode ---------------------------
    xb, _ = pipeline.synthetic_batch(n, seed=1, device="cuda", channels_last=True)
    base = dict(pipeline.CONFIGS["resnet50_w4a4"], clipping="mse", stats_mode="collect")
    step = {False: [], True: []}
    fps = {"gaus": [], "mse": []}
    with tempfile.TemporaryDirectory() as tmp:
        # the per-tensor statistics use mode reads too
        m0, q0 = pipeline.build_quantized_model(dict(base, per_channel_quant_act=False, bit_alloc_act=False,
                                                     stats_folder="joint", stats_base_dir=tmp), "cuda", channels_last=True)
        with torch.no_grad():
            m0(xb)
        q0.__exit__()
        q0.detach()
        del m0
        models = {}
        for on in (False, True):
            cfg = dict(base, stats_folder="joint" if on else "curves", stats_base_dir=tmp, collect_mse=True, collect_bits=on)
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
            models[on][1].__exit__()   # the "joint" folder: statistics of 2 + 2 * rounds batches, curves and tables
            models[on][1].detach()
        del models
        torch.cuda.empty_cache()
        use = {}
        for prior in ("gaus", "mse"):
            cfg = dict(pipeline.CONFIGS["resnet50_w4a4"], clipping="mse", stats_mode="use", stats_folder="joint",
                       stats_base_dir=tmp, bit_alloc_prior=prior)
            use[prior] = pipeline.build_quantized_model(cfg, "cuda", channels_last=True)
        logits = {}
        with torch.no_grad():
            for prior in ("gaus", "mse"):
                logits[prior] = use[prior][0](xb)
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            for _ in range(a.rounds):
                for prior in ("gaus", "mse"):
                    ev[0].record()
                    for _ in range(5):
                        use[prior][0](xb)
                    ev[1].record()
                    torch.cuda.synchronize()
                    fps[prior].append(5 * n / (ev[0].elapsed_time(ev[1]) * 1e-3))
        finite = all(bool(torch.isfinite(v).all()) for v in logits.values())
        for prior in ("gaus", "mse"):
            use[prior][1].detach()
    r = prof["modes"].get("R", {"launches": 0, "ms": 0.0, "elems": 0})
    off, on = median(step[False]), median(step[True])
    res = {
        "tool": "joint_mse_bench", "gpu": gpu_info(), "shape": [n, 64, 112, 112], "num_bits": 4, "widths": widths,
        "multipliers": len(MSE_MULTIPLIERS),
        "clip_mse_grid": {"ms_median": round(ms_grid, 1), "candidate_evaluations_per_s": float("%.3g" % (evals / (ms_grid * 1e-3))),
                          "five_clip_mse_launches_ms_median": round(ms_split, 1), "columns_equal": same},
        "resnet50_w4a4_collect_c_mse_channels_last": {
            "batch": n, "rounds": a.rounds, "s_per_batch_collect_mse": round(off, 3),
            "s_per_batch_collect_mse_and_bits": round(on, 3),
            "s_per_batch_collect_mse_all": [round(v, 3) for v in step[False]],
            "s_per_batch_collect_mse_and_bits_all": [round(v, 3) for v in step[True]],
            "clip_mse_launches": r["launches"], "clip_mse_gpu_ms": round(r["ms"], 1)},
        "resnet50_w4a4_use_c_mse_channels_last": {
            "batch": n, "images_per_s_baa": round(median(fps["gaus"])), "images_per_s_baa_bap_mse": round(median(fps["mse"])),
            "images_per_s_baa_all": [round(v) for v in fps["gaus"]],
            "images_per_s_baa_bap_mse_all": [round(v) for v in fps["mse"]], "logits_finite": finite},
        "note": "kernel times are CUDA events around each call; collect steps are host-clock times around synchronised "
                "forwards; use-mode rates are CUDA events around 5 forwards",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    c, u = res["resnet50_w4a4_collect_c_mse_channels_last"], res["resnet50_w4a4_use_c_mse_channels_last"]
    print("| `h100_joint_mse_bench.json` | `python tools/joint_mse_bench.py`: the cost of `-c mse -bap mse`. Taken on %s. "
          "`ops.clip_mse_grid` (9 widths x 125 multipliers) on %dx64x112x112 channels-last: %.1f ms (%.3g candidate "
          "evaluations/s); the five `ops.clip_mse(widths=...)` launches over the same pairs %.1f ms, columns equal: %s. "
          "ResNet-50 W4A4 `-sm collect -c mse` at batch %d, channels-last: %.2f s per batch with collect_mse, %.2f s with "
          "collect_mse + collect_bits (%d clip_mse launches, %.0f ms GPU). `-sm use -c mse -baa`: %d images/s, with "
          "`-bap mse` %d |"
          % (res["gpu"], n, ms_grid, evals / (ms_grid * 1e-3), ms_split, same, n, off, on, c["clip_mse_launches"],
             c["clip_mse_gpu_ms"], u["images_per_s_baa"], u["images_per_s_baa_bap_mse"]))


if __name__ == "__main__":
    main()
