#!/usr/bin/env python
"""Every quantized cell of the paper's results table (``pipeline.PAPER_TABLE``: 8W4A, 4W8A and 4W4A rows on the six
networks) through the REAL reference manager (class swap + quantize_model + one forward on CPU), batch 2 at small crops.

What is kept, in compact form (tests/golden/ref_census_paper_table.json / ref_pipeline_paper_table.npz):
* the call list of every quantize_instant (id, tag, half_range, shape) depends on the network only: the run checks that
  all cells of a network give the same list, and that it equals the list of that network's cell in ref_census.json /
  ref_census_paper_nets.json where one exists (the lists are not stored twice).  ResNet-101's, which no fixture has, is
  stored here;
* the ids of the weights quantized with the 8-bit attribute override (the first layers), per network;
* per cell, the first 32 of the 1000 logits of each sample, keyed "net|setting|method".

Build container only (needs the reference checkout).  Same set-up as make_census.py (its import does it); the models are
prepared as inference_sim.py:175-181 does (ResNets: before-relu marks and BN folding; VGG-16-BN and Inception-v3: BN
folding), Inception-v3 with the constructor keywords of ``pipeline.ARCH_KWARGS``.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_census as mc  # noqa: E402  (sets up the reference import, stubs and the CPU leaf)

sys.path.insert(0, mc.ROOT)
from cnn_quantization_b200.pipeline import ARCH_KWARGS, PAPER_TABLE  # noqa: E402

BATCH = 2
HW = {"inception_v3": 107}   # the smallest crops the networks take comfortably; 64 for the others
LOGITS = 32                  # logits kept per sample
# the existing census entry of each network (same batch and crop), whose call list the table's cells must reproduce
KNOWN = {"resnet18": ("ref_census.json", "resnet18_w4a4"), "resnet50": ("ref_census.json", "resnet50_w4a4"),
         "vgg16": ("ref_census.json", "vgg16_w4a4"), "inception_v3": ("ref_census_paper_nets.json", "inception_v3_w4a4"),
         "vgg16_bn": ("ref_census_paper_nets.json", "vgg16_bn_w4a4")}


def key(cell):
    return "|".join(cell)


def run(cell):
    from itertools import count
    flags = dict(PAPER_TABLE[cell])
    arch = flags.pop("arch")
    hw = HW.get(arch, 64)
    mc.Singleton._instances.clear()
    for cls in (mc.iqm.Conv2dWithId, mc.iqm.LinearWithId, mc.iqm.MaxPool2dWithId, mc.iqm.AvgPool2dWithId, mc.iqm.BatchNorm2dWithId):
        cls._id = count(0)
    args = mc.make_args(arch=arch, **flags)
    calls = []
    orig = mc.iqm.TruncationOpManagerInference.quantize_instant

    def spy(self, tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False):
        calls.append([id, tag, bool(half_range), list(tensor.shape), list(override_att) if override_att else None])
        return orig(self, tensor, id, tag, stat_id, half_range, override_att, False)

    mc.iqm.TruncationOpManagerInference.quantize_instant = spy
    try:
        with mc.iqm.QuantizationManagerInference(args, mc.qparams(args)) as qm:
            torch.manual_seed(12345)
            model = mc.models.__dict__[arch](weights=None, **ARCH_KWARGS.get(arch, {}))
            mc.set_node_names(model)
            if "resnet" in arch:
                mc.resnet_mark_before_relu(model)
            if "resnet" in arch or arch in ("vgg16_bn", "inception_v3"):
                mc.search_absorbe_bn(model)
                qm.bn_folding = True
            model.eval()
            qm.quantize_model(model)
            n_weight_calls = len(calls)
            rs = np.random.RandomState(12345)
            x = torch.from_numpy(rs.standard_normal((BATCH, 3, hw, hw)).astype(np.float32))
            with torch.no_grad():
                y = model(x)
    finally:
        mc.iqm.TruncationOpManagerInference.quantize_instant = orig
    return dict(weight_calls=calls[:n_weight_calls], act_calls=calls[n_weight_calls:], hw=hw, batch=BATCH,
                flags=PAPER_TABLE[cell]), y.numpy()


def write(results):
    """``results``: {cell: (census entry of run(), logits)} -> the two fixture files."""
    census = {"batch": BATCH, "hw": {}, "first8": {}, "calls": {}, "known": {n: list(v) for n, v in KNOWN.items()}}
    logits = {}
    for cell, (c, y) in results.items():
        net = cell[0]
        calls = [[k[:4] for k in c["weight_calls"]], [k[:4] for k in c["act_calls"]]]
        first8 = [k[0] for k in c["weight_calls"] if k[4] == ["num_bits", 8]]
        if net in census["hw"]:   # every cell of a network makes the same calls
            assert (census["hw"][net], census["first8"][net], census["calls"].get(net, calls)) == (c["hw"], first8, calls), cell
            if net in KNOWN:
                assert calls == known_calls(net), cell
        else:
            census["hw"][net], census["first8"][net] = c["hw"], first8
            if net in KNOWN:
                assert calls == known_calls(net), cell
            else:
                census["calls"][net] = calls
        logits[key(cell)] = np.ascontiguousarray(y[:, :LOGITS])
    with open(os.path.join(HERE, "ref_census_paper_table.json"), "w") as f:
        json.dump(census, f)
    np.savez_compressed(os.path.join(HERE, "ref_pipeline_paper_table.npz"), **logits)


def known_calls(net):
    fname, name = KNOWN[net]
    with open(os.path.join(HERE, fname)) as f:
        e = json.load(f)[name]
    return [e["weight_calls"], e["act_calls"]]


def main():
    torch.set_num_threads(8)
    results = {}
    for cell in PAPER_TABLE:
        if PAPER_TABLE[cell].get("q_off"):
            continue   # the FP32 column quantizes nothing
        results[cell] = run(cell)
        print(key(cell), len(results[cell][0]["weight_calls"]), "weight calls,", len(results[cell][0]["act_calls"]),
              "activation calls", flush=True)
    write(results)


if __name__ == "__main__":
    main()
