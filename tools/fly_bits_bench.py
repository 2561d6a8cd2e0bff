#!/usr/bin/env python
"""The cost of `-baa -bap mse` on the fly (`-sm no`, fly_bits), timed on the GPU.  Writes one JSON object (--out) and
prints it, followed by the row profiles/README.md keeps for it.

  * ResNet-50 W4A4 (`-pcq_w -pcq_a -baa -baw -bcw`) on channels-last memory at batch 512, in images per second, with
    `-c laplace` (analytic widths), fly_bits under `-c laplace`, and fly_bits under `-c mse` at 33 multipliers (2.0 ..
    10.0 in steps of 0.25), alternated round by round in the same process (host clock around a synchronised forward);
  * the GPU time of one forward of each, per launch mode of the ops launch profile (CUDA events; 'S' the statistics-only
    launches, 'R' the candidate sums, 'L' the allocations, 'A' the given-parameter applies);
  * the allocator alone on random [G, 9] tables at G = 2048, target 4, and at ResNet-50's 53 allocated channel counts:
    fqb200_allocate_widths of this library against the same entry of a library built from an earlier source tree
    (--parent-lib; `tools/build_parent_lib.sh <revision>` builds one with build.py's flags, by default from HEAD~1),
    alternated, CUDA events.  Without that library the comparison is skipped and the JSON says so.
The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys
import time

from benchlib import ROOT, build_or_exit, gpu_info, median, timed, write_json

# ResNet-50's allocated activation call sites: channel counts and how many there are
RESNET50_GROUPS = ((64, 7), (128, 8), (256, 16), (512, 11), (1024, 7), (2048, 4))


def _allocator(lib_path):
    """fqb200_allocate_widths(sse, target) -> widths of the library at ``lib_path`` (its own ctypes handle)."""
    import torch
    from cnn_quantization_b200 import _lib as L
    lib = ctypes.CDLL(lib_path)
    for name in ("fqb200_allocate_widths", "fqb200_allocate_widths_workspace_bytes"):
        restype, argtypes = L.PROTOTYPES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = restype, argtypes
    ws = {}

    def run(sse, target):
        g = sse.shape[0]
        key = (g, target)
        if key not in ws:
            ws[key] = torch.empty(lib.fqb200_allocate_widths_workspace_bytes(g, float(target)), dtype=torch.uint8,
                                  device=sse.device)
        out = torch.empty(g, dtype=torch.float32, device=sse.device)
        L.check(lib.fqb200_allocate_widths(sse.data_ptr(), g, float(target), out.data_ptr(), None, ws[key].data_ptr(),
                                           ws[key].numel(), torch.cuda.current_stream().cuda_stream))
        return out
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent-lib", default=os.path.join(ROOT, "tools", "_variants", "libfqb200_parent.so"))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fly_bits_bench.json"))
    a = ap.parse_args()
    build_or_exit("fly_bits_bench.py")
    import numpy as np
    import torch
    from cnn_quantization_b200 import _lib as L, pipeline

    # -- the allocator alone: this library against the parent's ----------------------------------------------------------
    libs = {"new": _allocator(L.LIB_PATH)}
    if os.path.exists(a.parent_lib):
        libs["parent"] = _allocator(a.parent_lib)
    else:
        sys.stderr.write("fly_bits_bench: no library at %s (tools/build_parent_lib.sh builds one): the parent allocator "
                         "is not measured\n" % a.parent_lib)
    rs = np.random.RandomState(0)

    def table(g):
        return torch.from_numpy(np.sort(rs.gamma(0.5, 1.0, (g, 9)), 1)[:, ::-1] * rs.uniform(0.1, 10.0, (g, 1))).cuda()

    alloc = {}
    t2048 = table(2048)
    same = True
    ms = {k: [] for k in libs}
    for k, fn in libs.items():
        fn(t2048, 4)
    for _ in range(a.reps):
        for k, fn in libs.items():
            ms[k] += timed(lambda: fn(t2048, 4))
    if "parent" in libs:
        same = bool(torch.equal(libs["new"](t2048, 4), libs["parent"](t2048, 4)))
    alloc["G2048_target4_ms"] = {k: round(median(v), 3) for k, v in ms.items()}
    tables = [(g, table(g)) for g, count in RESNET50_GROUPS for _ in range(count)]
    per_forward = {}
    for k, fn in libs.items():
        for g, t in tables:
            fn(t, 4)
    for k in libs:
        per_forward[k] = []
    for _ in range(a.reps):
        for k, fn in libs.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for g, t in tables:
                fn(t, 4)
            e1.record()
            torch.cuda.synchronize()
            per_forward[k].append(e0.elapsed_time(e1))
    if "parent" in libs:
        same = same and all(torch.equal(libs["new"](t, 4), libs["parent"](t, 4)) for _, t in tables)
    alloc["resnet50_53_tables_target4_ms"] = {k: round(median(v), 3) for k, v in per_forward.items()}
    alloc["widths_identical_to_parent"] = same if "parent" in libs else "parent library not given: not measured"
    del t2048, tables
    torch.cuda.empty_cache()

    # -- ResNet-50 W4A4, channels-last, batch 512 ----------------------------------------------------------------------
    n = a.batch
    short = [2.0 + 0.25 * i for i in range(33)]
    runs = {"laplace": dict(clipping="laplace"),
            "fly_bits_laplace": dict(clipping="laplace", bit_alloc_prior="mse", fly_bits=True),
            "fly_bits_mse_k33": dict(clipping="mse", bit_alloc_prior="mse", fly_bits=True, mse_multipliers=short)}
    xb, _ = pipeline.synthetic_batch(n, seed=1, device="cuda", channels_last=True)
    models = {k: pipeline.build_quantized_model(dict(pipeline.CONFIGS["resnet50_w4a4"], **v), "cuda", channels_last=True)
              for k, v in runs.items()}
    from cnn_quantization_b200 import ops
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
        "tool": "fly_bits_bench", "gpu": gpu_info(), "batch": n,
        "flags": "-pcq_w -pcq_a -baa -baw -bcw, int4, channels-last; fly_bits runs add -bap mse",
        "multipliers_k33": [short[0], short[-1], 0.25],
        "resnet50_w4a4": net,
        "allocator": alloc,
        "note": "images/s from host-clock times around a synchronised forward, the three configurations alternated round "
                "by round; GPU times per launch mode from CUDA events in a separate profiled forward; allocator times are "
                "CUDA-event medians on random tables, this library and the parent's alternated",
    }
    write_json(res, a.out)
    print(json.dumps(res))
    r = res["resnet50_w4a4"]
    fl = r["fly_bits_laplace"]["gpu_ms_per_mode"]
    print("| `h100_fly_bits_bench.json` | `python tools/fly_bits_bench.py`: `-baa -bap mse` on the fly (fly_bits). Taken on "
          "%s. ResNet-50 W4A4 (`-baa -baw -bcw`) at batch %d, channels-last: %.0f images/s with `-c laplace`, %.0f with "
          "fly_bits, %.0f with fly_bits `-c mse` at 33 multipliers; per fly_bits forward 'L' %.1f ms against 'R' %.1f ms. "
          "Allocator at G = 2048, target 4: %s ms (new / parent) |"
          % (res["gpu"], n, r["laplace"]["images_per_s"], r["fly_bits_laplace"]["images_per_s"],
             r["fly_bits_mse_k33"]["images_per_s"], fl.get("L", {}).get("gpu_ms", float("nan")),
             fl.get("R", {}).get("gpu_ms", float("nan")),
             " / ".join(str(v) for v in alloc["G2048_target4_ms"].values())))


if __name__ == "__main__":
    main()
