#!/usr/bin/env python
"""Throughput of the two paper networks added with their launch fusions, on the GPU.  Writes one JSON object (--out) and
prints it.

For inception_v3_w4a4 (299x299) and vgg16_bn_w4a4 (224x224), channels-last, batch --batch, one seeded model per arm:
  * "fused": the manager as it ships - Inception branches write into their block's output (no torch.cat), the functional
    ReLU of BasicConv2d is skipped, VGG-16-BN's poolings run inside the quantization launches;
  * "unfused": the same model without what this tool measures (``OFF``, manager attributes): for Inception-v3 the slice
    writes and the BasicConv2d ReLU skip (``skip_redundant_relu`` gates nothing else there: the network has no nn.ReLU
    module); for VGG-16-BN only the in-launch pooling - its hooked nn.ReLU modules are skipped in both arms, as before;
both arms warmed up, then --rounds rounds of --steps forwards each, alternating A B B A, timed with CUDA events around
the forwards (images/s = batch * steps / time).  The logits of both arms on the timed batch must be equal (torch.equal).
"""
import argparse
import json
import os

import numpy as np

from benchlib import ROOT, build_or_exit, gpu_info, timed, write_json

OFF = {"inception_v3_w4a4": ("fuse_inception_concat", "skip_redundant_relu"), "vgg16_bn_w4a4": ("fuse_pool_into_quant",)}


def build(config, fused):
    from cnn_quantization_b200 import pipeline
    model, qm = pipeline.build_quantized_model(config, "cuda", channels_last=True)
    if not fused:
        qm.detach()
        for attr in OFF[config]:
            setattr(qm, attr, False)
        qm.attach(model)
    return model, qm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_paper_nets_bench.json"))
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--configs", default="inception_v3_w4a4,vgg16_bn_w4a4")
    a = ap.parse_args()
    build_or_exit("paper_nets_bench.py")
    import torch
    from cnn_quantization_b200 import pipeline
    res ={"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "batch": a.batch, "steps": a.steps,
           "warmup": a.warmup, "rounds": a.rounds, "memory_format": "channels_last", "configs": {}}
    for config in a.configs.split(","):
        hw = pipeline.INPUT_SIZE[config]
        x, _ = pipeline.synthetic_batch(a.batch, seed=7, channels_last=True, config=config)
        x = x.cuda().contiguous(memory_format=torch.channels_last)
        arms = {"fused": build(config, True), "unfused": build(config, False)}
        logits = {}
        with torch.no_grad():
            for name, (model, _) in arms.items():
                for _ in range(a.warmup):
                    model(x)
                logits[name] = model(x).clone()
            times = {k: [] for k in arms}
            for r in range(a.rounds):
                for name in (("fused", "unfused", "unfused", "fused") if r % 2 == 0 else ("unfused", "fused", "fused", "unfused")):
                    model = arms[name][0]
                    times[name].append(timed(lambda: [model(x) for _ in range(a.steps)])[0] / 1e3)
        entry = {"hw": hw, "unfused_arm_disables": list(OFF[config]),
                 "logits_equal": bool(torch.equal(logits["fused"], logits["unfused"]))}
        for name, ts in times.items():
            rates = [a.batch * a.steps / t for t in ts]
            entry[name] = {"images_per_s_median": float(np.median(rates)), "images_per_s_all": rates}
        entry["speedup"] = entry["fused"]["images_per_s_median"] / entry["unfused"]["images_per_s_median"]
        res["configs"][config] = entry
        print(config, json.dumps(entry), flush=True)
        for model, qm in arms.values():
            qm.detach()
        del arms, x, logits
        torch.cuda.empty_cache()
    write_json(res, a.out)
    print(json.dumps(res))
    if not all(e["logits_equal"] for e in res["configs"].values()):
        raise SystemExit("fused and unfused logits differ")


if __name__ == "__main__":
    main()
