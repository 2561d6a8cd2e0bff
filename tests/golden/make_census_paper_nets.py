#!/usr/bin/env python
"""The two networks of the paper's table that ``ref_census.json`` does not cover, Inception-v3 and VGG-16-BN, through the
REAL reference manager (class swap + quantize_model + one forward on CPU): every quantize_instant call and the logits ->
tests/golden/ref_census_paper_nets.json / ref_pipeline_paper_nets.npz.

Build container only (needs the reference checkout).  Same set-up as make_census.py (its import does it); both networks
are BN-folded as inference_sim.py:179 does, and Inception-v3 is constructed with the keyword arguments
``pretrained=True`` uses (``pipeline.ARCH_KWARGS``) without loading the checkpoint.
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
from cnn_quantization_b200.pipeline import ARCH_KWARGS  # noqa: E402

W4A4 = dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
            bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)
CONFIGS = {
    # name: (arch, input hw, batch, flags)
    "inception_v3_w4a4": ("inception_v3", 107, 2, W4A4),
    "vgg16_bn_w4a4": ("vgg16_bn", 64, 2, W4A4),
}


def run(name):
    from itertools import count
    arch, hw, batch, flags = CONFIGS[name]
    mc.Singleton._instances.clear()
    for cls in (mc.iqm.Conv2dWithId, mc.iqm.LinearWithId, mc.iqm.MaxPool2dWithId, mc.iqm.AvgPool2dWithId, mc.iqm.BatchNorm2dWithId):
        cls._id = count(0)
    args = mc.make_args(arch=arch, **flags)
    calls = []
    orig = mc.iqm.TruncationOpManagerInference.quantize_instant

    def spy(self, tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False):
        calls.append([id, tag, bool(half_range), list(tensor.shape)])
        return orig(self, tensor, id, tag, stat_id, half_range, override_att, False)

    mc.iqm.TruncationOpManagerInference.quantize_instant = spy
    try:
        with mc.iqm.QuantizationManagerInference(args, mc.qparams(args)) as qm:
            torch.manual_seed(12345)
            model = mc.models.__dict__[arch](weights=None, **ARCH_KWARGS.get(arch, {}))
            mc.set_node_names(model)
            mc.search_absorbe_bn(model)   # inference_sim.py:177-181: vgg16_bn and inception_v3 are BN-folded
            qm.bn_folding = True
            model.eval()
            qm.quantize_model(model)
            n_weight_calls = len(calls)
            rs = np.random.RandomState(12345)
            x = torch.from_numpy(rs.standard_normal((batch, 3, hw, hw)).astype(np.float32))
            with torch.no_grad():
                y = model(x)
    finally:
        mc.iqm.TruncationOpManagerInference.quantize_instant = orig
    return dict(weight_calls=calls[:n_weight_calls], act_calls=calls[n_weight_calls:]), y.numpy()


def main():
    torch.set_num_threads(8)
    census, logits = {}, {}
    for name in CONFIGS:
        c, y = run(name)
        c.update(arch=CONFIGS[name][0], hw=CONFIGS[name][1], batch=CONFIGS[name][2], flags=CONFIGS[name][3])
        census[name] = c
        logits[name] = y
        print(name, len(c["weight_calls"]), "weight calls,", len(c["act_calls"]), "activation calls")
    with open(os.path.join(HERE, "ref_census_paper_nets.json"), "w") as f:
        json.dump(census, f)
    np.savez_compressed(os.path.join(HERE, "ref_pipeline_paper_nets.npz"), **logits)


if __name__ == "__main__":
    main()
