#!/usr/bin/env python
"""Throughput of every cell of the paper's results table (``pipeline.PAPER_TABLE``: 8W4A, 4W8A, 4W4A rows and the FP32
column on six networks) on the GPU.  Writes one JSON object (--out) and prints one line per cell.

Each cell: one seeded model (``pipeline.build_paper_cell``), channels-last, batch --batch at the cell's crop (299 for
Inception-v3, 224 otherwise), --warmup forwards, then --steps forwards timed with CUDA events (images/s = batch * steps /
time).  Inception-v3's 4W8A cells, whose per-tensor int8 branch outputs the per-sample min-max launch now writes straight
into the block's output, are also run with ``fuse_inception_concat`` off (``torch.cat`` of the branch outputs): both arms
of such a cell are timed --rounds times, alternating A B B A, and their logits on the timed batch must be equal.
"""
import argparse
import json
import os
import subprocess

import numpy as np

from benchlib import ROOT, build_or_exit, gpu_info, timed, write_json


def sm_clocks():
    """'max SM clock, current SM clock' of the first GPU as nvidia-smi reports them (read right after a timed cell), or
    'unknown'."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_paper_table_bench.json"))
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--nets", default="", help="comma-separated subset of pipeline.PAPER_NETS (default: all)")
    a = ap.parse_args()
    build_or_exit("paper_table_bench.py")
    import torch
    from cnn_quantization_b200 import pipeline
    nets = a.nets.split(",") if a.nets else list(pipeline.PAPER_NETS)
    res = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "batch": a.batch, "steps": a.steps,
           "warmup": a.warmup, "rounds": a.rounds, "memory_format": "channels_last", "cells": {},
           "inception_concat": {}}
    inputs = {}
    for cell in pipeline.PAPER_TABLE:
        if cell[0] not in nets:
            continue
        hw = pipeline.paper_cell_input_size(cell)
        if hw not in inputs:
            x, _ = pipeline.synthetic_batch(a.batch, seed=7, channels_last=True, hw=hw)
            inputs[hw] = x.cuda().contiguous(memory_format=torch.channels_last)
        x = inputs[hw]
        both = cell[0] == "inception_v3" and cell[1] == "4W8A"
        arms = {"on": pipeline.build_paper_cell(cell, "cuda", channels_last=True)}
        if both:
            model, qm = pipeline.build_paper_cell(cell, "cuda", channels_last=True)
            qm.detach()
            qm.fuse_inception_concat = False
            qm.attach(model)
            arms["off"] = (model, qm)
        logits, times = {}, {k: [] for k in arms}
        with torch.no_grad():
            for name, (model, _) in arms.items():
                for _ in range(a.warmup):
                    model(x)
                logits[name] = model(x).clone()
            order = [("on", "off", "off", "on") if r % 2 == 0 else ("off", "on", "on", "off") for r in range(a.rounds)] if both \
                else [("on",)]
            for names in order:
                for name in names:
                    model = arms[name][0]
                    times[name].append(timed(lambda: [model(x) for _ in range(a.steps)])[0] / 1e3)
        clocks = sm_clocks()
        rates = {k: [a.batch * a.steps / t for t in ts] for k, ts in times.items()}
        key = "|".join(cell)
        res["cells"][key] = {"hw": hw, "images_per_s": float(np.median(rates["on"])), "images_per_s_all": rates["on"],
                             "logits_finite": bool(torch.isfinite(logits["on"]).all()), "sm_clocks_after": clocks}
        if both:
            entry = {"concat_on": {"images_per_s_median": float(np.median(rates["on"])), "images_per_s_all": rates["on"]},
                     "concat_off": {"images_per_s_median": float(np.median(rates["off"])), "images_per_s_all": rates["off"]},
                     "logits_equal": bool(torch.equal(logits["on"], logits["off"]))}
            entry["speedup"] = entry["concat_on"]["images_per_s_median"] / entry["concat_off"]["images_per_s_median"]
            res["inception_concat"][key] = entry
        print(key, json.dumps(res["cells"][key]), json.dumps(res["inception_concat"].get(key, {})), flush=True)
        for model, qm in arms.values():
            qm.detach()
        del arms, logits
        torch.cuda.empty_cache()
    write_json(res, a.out)
    if not all(e["logits_equal"] for e in res["inception_concat"].values()):
        raise SystemExit("logits with and without fuse_inception_concat differ")
    if not all(e["logits_finite"] for e in res["cells"].values()):
        raise SystemExit("a cell gave non-finite logits")


if __name__ == "__main__":
    main()
