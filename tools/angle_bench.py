#!/usr/bin/env python
"""The cost of the sample-angle measurement (`-ms` with measure_stats_kind="angle"), timed on the GPU.  Writes one JSON
object (--out) and prints it, followed by the row profiles/README.md keeps for it.

  * ResNet-50 W4A4 (BASELINE configs[2]) channels-last at batch 512, inputs resident: the CUDA-event time of all
    ops.sample_angles launches of one forward (profile mode 'G'), and the FP64 rate they reach: (N (N + 1) / 2) * D
    multiply-adds per measured tensor, from the shapes, over that time, against the H100 SXM data sheet's 67 TFLOP/s FP64
    (tensor core).  FP64 compute bounds this work: its data is read once (4 B/element).
  * images/s with the angle kind on, the norm kind on and measurement off, alternated round by round in one process, with
    the logits checked equal across the three arms;
  * the reference's per-pair loop (acos(cos_sim(t[i], t[j])) with a float() per pair) written out here, timed on a few
    hundred pairs of the stem output and extrapolated to every pair of one forward (an extrapolation, not a run).
Writing angle.pkl (once per run) is not measured.
"""
import argparse
import json
import os
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json

FP64_PEAK = 67e12   # H100 SXM data sheet, FP64 tensor core, FLOP/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2, help="forwards per arm per round")
    ap.add_argument("--pairs", type=int, default=300, help="pairs of the reference's loop timed")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_angle_bench.json"))
    a = ap.parse_args()
    build_or_exit("angle_bench.py")
    import torch
    from cnn_quantization_b200 import ops, pipeline
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gpu = gpu_info()

    cfg = pipeline.CONFIGS["resnet50_w4a4"]
    xb, _ = pipeline.synthetic_batch(a.batch, seed=1, device="cuda", channels_last=True)
    arms = {"off": dict(cfg), "distance": dict(cfg, measure_stats=True),
            "angle": dict(cfg, measure_stats=True, measure_stats_kind="angle")}
    models = {k: pipeline.build_quantized_model(v, "cuda", channels_last=True) for k, v in arms.items()}
    logits = {}
    with torch.no_grad():
        for k, (model, qm) in models.items():
            logits[k] = model(xb).clone()
            if qm.measure_stats is not None:
                qm.measure_stats.stats = {}
        torch.cuda.synchronize()
        rates = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, (model, qm) in models.items():
                t = timed(lambda: [model(xb) for _ in range(a.steps)])[0]
                rates[k].append(a.batch * a.steps / (t * 1e-3))
                if qm.measure_stats is not None:
                    qm.measure_stats.stats = {}   # keep only what one round measured
        # one profiled angle forward: the 'G' launches' event time and the shapes they ran on
        ops.profile_reset(enable=True)
        models["angle"][0](xb)
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
    equal = all(torch.equal(logits["off"], logits[k]) for k in ("distance", "angle"))
    g = prof["modes"].get("G", {"launches": 0, "ms": 0.0, "elems": 0})
    fma = 0
    for key, v in prof["shapes"].items():
        if key.startswith("G "):
            n, d = (int(s) for s in key[2:].split("x"))
            fma += v["launches"] * n * (n + 1) // 2 * d
    flops = 2.0 * fma / (g["ms"] * 1e-3) if g["ms"] else None

    # the reference's per-pair loop on the stem output (angle_stats.py:17-37 with utils/misc.py cos_sim), extrapolated
    with torch.no_grad():
        model, qm = models["distance"]   # the fusions that never write the measured tensor are off there
        stem = {}

        def keep(m, i, o):
            stem["t"] = o.detach().contiguous()

        h = model.conv1.register_forward_hook(keep)
        model(xb)
        h.remove()
        qm.measure_stats.stats = {}
        t = stem["t"].view(a.batch, -1)

        def ref_pair(x, y):
            cos = (x * y).sum(-1) / (torch.sqrt((x ** 2).sum(-1)) * torch.sqrt((y ** 2).sum(-1)))
            return float(torch.acos(cos))

        pairs = [(i, j) for i in range(a.batch) for j in range(i + 1, a.batch)][:a.pairs]
        for i, j in pairs[:10]:
            ref_pair(t[i], t[j])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i, j in pairs:
            ref_pair(t[i], t[j])
        per_pair_s = (time.perf_counter() - t0) / len(pairs)
    all_pairs = g["launches"] * a.batch * (a.batch - 1) // 2
    res = {
        "tool": "angle_bench", "gpu": gpu, "batch": a.batch,
        "sample_angles": {"launches": g["launches"], "ms": round(g["ms"], 2), "fma": fma,
                          "fp64_tflop_s": round(flops / 1e12, 2) if flops else None,
                          "fraction_of_67_tflop_s": round(flops / FP64_PEAK, 3) if flops else None,
                          "bound": "FP64 compute (each tensor is read once, 4 B/element)"},
        "resnet50_w4a4_cl": {"rounds": a.rounds, "steps_per_round": a.steps,
                             "images_per_s": {k: round(median(v), 1) for k, v in rates.items()},
                             "images_per_s_all": {k: [round(x, 1) for x in v] for k, v in rates.items()},
                             "logits_equal_across_arms": equal},
        "reference_loop_extrapolated": {"pairs_timed": len(pairs), "tensor": "stem output %dx%d" % tuple(t.shape),
                                        "s_per_pair": round(per_pair_s, 7), "pairs_per_forward": all_pairs,
                                        "s_per_forward_extrapolated": round(per_pair_s * all_pairs, 1)},
        "note": "FP64 rate = 2 * sum(N (N + 1) / 2 * D) over the 'G' launches' event time of one profiled forward, against "
                "the 67 TFLOP/s data-sheet figure; the reference loop is timed on the stem output only and extrapolated "
                "to every pair of every measured tensor at that per-pair cost (not run end to end); angle.pkl is not "
                "written or timed",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    s, r = res["sample_angles"], res["resnet50_w4a4_cl"]["images_per_s"]
    print("| `h100_angle_bench.json` | `python tools/angle_bench.py`: the angle kind of `-ms`. Taken on %s. ResNet-50 W4A4 "
          "channels-last at batch %d: %d `sample_angles` launches %.1f ms per forward, %.1f TFLOP/s FP64 (%.2f of 67, "
          "FP64-compute bound); %.0f images/s off, %.0f with the norm kind, %.0f with the angle kind |"
          % (gpu, a.batch, s["launches"], s["ms"], s["fp64_tflop_s"] or 0, s["fraction_of_67_tflop_s"] or 0, r["off"],
             r["distance"], r["angle"]))
    if not equal:
        raise SystemExit("logits differ across the arms")


if __name__ == "__main__":
    main()
