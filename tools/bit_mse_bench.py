#!/usr/bin/env python
"""The cost of measured bit allocation (collect_bits, `-bap mse`), timed on the GPU.  Writes one JSON object (--out) and
prints it, followed by the row profiles/README.md keeps for it.

  * ops.clip_mse with widths 0..8 (K = 9, the Laplace rule, positive) per channel on a 512 x 64 x 112 x 112
    channels-last tensor (the ResNet-50 stem output at batch 512, the largest tensor of the network): CUDA events around
    each call after a warm-up, against the one-read HBM bound (4 B/element at the H100 SXM data sheet's 3.35 TB/s), and
    against nine K = 1 launches (one width each) on the same tensor;
  * one ResNet-50 W4A4 `-sm collect` step on channels-last memory at batch 512, with and without collect_bits,
    alternated round by round in the same process (host clock around a synchronised forward);
  * the host time of bit_alloc.allocate on the largest layer's table (2048 channels, target 4), and ResNet-50
    quantize_model with `-baw -bap mse` against the analytic `-baw` (host clock around a synchronised call).
Writing the table files (once per run) is not measured.
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bit_mse_bench.json"))
    a = ap.parse_args()
    build_or_exit("bit_mse_bench.py")
    import numpy as np
    import torch
    from cnn_quantization_b200 import manager as M, ops, pipeline
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import bit_candidates

    # -- the kernel alone ------------------------------------------------------------------------------------------------
    n = a.batch
    x = torch.randn(n, 64, 112, 112, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    x = torch.relu(x).contiguous(memory_format=torch.channels_last)
    layout = (n, 64, 112 * 112)
    t_hbm = 4.0 * x.numel() / HBM_PEAK
    table = ops.fused(x, layout, stats_only=True, channels_last=True)
    mults, prior = bit_candidates("laplace", True, 4)
    mult = torch.tensor(mults, dtype=torch.float32, device="cuda")
    widths = list(range(9))
    k9 = lambda: ops.clip_mse(x, table, layout, True, 4, True, mult, prior=prior, widths=widths, solve_f64=False)
    singles = [(mult[w:w + 1], [w]) for w in widths]
    k1 = lambda: [ops.clip_mse(x, table, layout, True, 4, True, m, prior=prior, widths=w, solve_f64=False) for m, w in singles]
    k9(), k1()
    torch.cuda.synchronize()
    ms9 = median(timed(k9, a.reps))
    ms1 = median(timed(k1, a.reps))
    nine, ones = k9(), k1()
    same = all(torch.equal(nine[:, 1 + w], ones[w][:, 1]) for w in widths)
    del nine, ones
    del x, table
    torch.cuda.empty_cache()

    # -- allocate on the largest layer's table ---------------------------------------------------------------------------------
    rs = np.random.RandomState(0)
    big = np.sort(rs.random_sample((2048, 9)), axis=1)[:, ::-1] * rs.random_sample((2048, 1))
    allocate(big[:8], 4)
    t0 = time.perf_counter()
    allocate(big, 4)
    alloc_s = time.perf_counter() - t0

    # -- ResNet-50 quantize_model: -baw -bap mse against the analytic -baw (the second of two runs each) ------------------------
    qmodel = {}
    for prior_w in ("gaus", "mse") * 2:
        model, qm0 = pipeline.build_quantized_model(dict(arch="resnet50"), "cuda")   # fp32 weights, BN folded
        qm0.detach()
        args = M.make_args(**dict(pipeline.CONFIGS["resnet50_w4a4"], bit_alloc_prior=prior_w, bit_alloc_act=False))
        mgr = M.QuantizationManagerInference(args, M.get_params(args))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mgr.quantize_model(model)
        torch.cuda.synchronize()
        qmodel[prior_w] = time.perf_counter() - t0
        del model
    torch.cuda.empty_cache()

    # -- one ResNet-50 W4A4 collect step on channels-last memory, with and without collect_bits --------------------------------
    xb, _ = pipeline.synthetic_batch(n, seed=1, device="cuda", channels_last=True)
    step = {False: [], True: []}
    with tempfile.TemporaryDirectory() as tmp:
        models = {}
        for on in (False, True):
            cfg = dict(pipeline.CONFIGS["resnet50_w4a4"], stats_mode="collect", stats_folder="r50_%d" % on,
                       stats_base_dir=tmp, collect_bits=on)
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
        "tool": "bit_mse_bench", "gpu": gpu_info(), "shape": [n, 64, 112, 112], "num_bits": 4, "widths": widths,
        "bounds": {"hbm_read_ms": round(t_hbm * 1e3, 3)},
        "clip_mse_widths": {"k9_ms_median": round(ms9, 2), "fraction_of_hbm_bound": round(t_hbm / (ms9 * 1e-3), 3),
                            "nine_k1_launches_ms_median": round(ms1, 2), "columns_equal_k1": same},
        "allocate_2048x9_target4_s": round(alloc_s, 3),
        "resnet50_quantize_model_s": {"baw_analytic": round(qmodel["gaus"], 3), "baw_bap_mse": round(qmodel["mse"], 3)},
        "resnet50_w4a4_collect_channels_last": {
            "batch": n, "rounds": a.rounds, "s_per_batch_without": round(off, 3), "s_per_batch_with": round(on, 3),
            "s_per_batch_without_all": [round(v, 3) for v in step[False]],
            "s_per_batch_with_all": [round(v, 3) for v in step[True]],
            "clip_mse_launches": r["launches"], "clip_mse_gpu_ms": round(r["ms"], 1)},
        "note": "HBM bound from the H100 SXM data sheet (3.35 TB/s for one 4 B/element read), not measured; collect steps, "
                "allocate and quantize_model are host-clock times around synchronised work",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    c = res["resnet50_w4a4_collect_channels_last"]
    print("| `h100_bit_mse_bench.json` | `python tools/bit_mse_bench.py`: collect_bits / `-bap mse` cost. Taken on %s. "
          "`ops.clip_mse` with widths 0..8 (K = 9) on %dx64x112x112 channels-last: %.2f ms (%.2f of the %.2f ms one-read "
          "HBM bound), nine K = 1 launches %.2f ms. `allocate` on 2048 channels: %.3f s. ResNet-50 quantize_model %.2f s "
          "with `-baw -bap mse`, %.2f s with the analytic `-baw`. ResNet-50 W4A4 collect at batch %d, channels-last: %.2f s "
          "per batch without, %.2f s with collect_bits (%d clip_mse launches, %.0f ms GPU) |"
          % (res["gpu"], n, ms9, t_hbm / (ms9 * 1e-3), t_hbm * 1e3, ms1, alloc_s, qmodel["mse"], qmodel["gaus"], n, off, on,
             c["clip_mse_launches"], c["clip_mse_gpu_ms"]))


if __name__ == "__main__":
    main()
