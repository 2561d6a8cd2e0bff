#!/usr/bin/env python
"""Collect-mode KL-divergence calibration (`-kld -sm collect`) of every hooked ResNet-50 tensor at batch 512, timed on the
GPU.  Prints one JSON line.

The hooked tensors are the outputs of the convolutions, the linear layer and the two poolings (the manager's collect
hooks), shapes from torchvision's resnet50 at 224x224 on the meta device.  Each tensor is a view of one buffer of N(0, 1)
values.  Two runs:
  * CUDA events around every ops.kld_threshold call (the three launches), after a warm-up: the time of one calibration batch;
  * torch.profiler with CUDA activities (a separate run): the histogram phase (max |x| pass + histogram pass, 8 B/element)
    in Gelem/s and as a fraction of the H100 SXM data-sheet HBM3 bandwidth, and the threshold search in us per row.
The reference's per-sample CPU time (kld_threshold._get_optimal_threshold, 2001 bins, numpy/scipy; measured on a CPU
host, about 0.33 s per sample for any of 64x56x56, 256x14x14, 2048x7x7) is printed beside these, with the batch figure
it implies labelled as an extrapolation.
"""
import argparse
import json

from benchlib import build_or_exit, gpu_info, median, timed

HBM_PEAK = 3.35e12               # H100 SXM data sheet, bytes/s
REF_CPU_S_PER_SAMPLE = 0.33      # the reference's search per sample on a CPU host (measured, see the docstring)


def hooked_shapes(batch):
    import torch
    import torchvision
    shapes = []
    model = torchvision.models.resnet50(weights=None).to("meta")
    kinds = (torch.nn.Conv2d, torch.nn.Linear, torch.nn.MaxPool2d, torch.nn.AdaptiveAvgPool2d)
    for m in model.modules():
        if isinstance(m, kinds):
            m.register_forward_hook(lambda m, i, o: shapes.append(tuple(o.shape)))
    with torch.no_grad():
        model(torch.empty(batch, 3, 224, 224, device="meta"))
    return shapes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    build_or_exit("kld_bench.py")
    import torch
    from cnn_quantization_b200 import ops

    shapes = hooked_shapes(a.batch)
    numel = [int(torch.Size(s).numel()) for s in shapes]
    buf = torch.randn(max(numel), device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    xs = [buf[:n].view(s) for n, s in zip(numel, shapes)]
    rows = sum(s[0] for s in shapes)
    elems = sum(numel)

    for x in xs:   # warm-up: module load, shared-memory attributes
        ops.kld_threshold(x)
    torch.cuda.synchronize()
    batch_ms = timed(lambda: [ops.kld_threshold(x)[0].max() for x in xs], a.reps)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for x in xs:
            ops.kld_threshold(x)
        torch.cuda.synchronize()
    kern = {"absmax": 0.0, "hist": 0.0, "search": 0.0}
    for ev in prof.events():
        name = ev.name
        for k in kern:
            if "fq_kld_%s_kernel" % k in name:
                kern[k] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
    hist_ms = kern["absmax"] + kern["hist"]
    res = {
        "tool": "kld_bench", "gpu": gpu_info(), "model": "resnet50", "batch": a.batch, "hooked_tensors": len(shapes),
        "rows": rows, "elements": elems,
        "batch_ms_median": median(batch_ms), "batch_ms_all": [round(v, 3) for v in batch_ms],
        "hist_phase_ms": round(hist_ms, 3), "absmax_ms": round(kern["absmax"], 3), "hist_ms": round(kern["hist"], 3),
        "hist_phase_gelem_s": round(elems / (hist_ms * 1e-3) / 1e9, 2) if hist_ms else None,
        "hist_phase_hbm_fraction": round(8.0 * elems / (hist_ms * 1e-3) / HBM_PEAK, 3) if hist_ms else None,
        "search_ms": round(kern["search"], 3), "search_us_per_row": round(kern["search"] * 1e3 / rows, 2),
        "ref_cpu_s_per_sample_measured": REF_CPU_S_PER_SAMPLE,
        "ref_cpu_batch_s_extrapolated": round(REF_CPU_S_PER_SAMPLE * rows, 1),
        "note": "ref_cpu_batch_s_extrapolated = measured per-sample CPU time x rows, not measured end to end; "
                "hbm fraction against the 3.35 TB/s data sheet, 8 B/element (two reads)",
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
