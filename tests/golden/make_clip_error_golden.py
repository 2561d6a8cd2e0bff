#!/usr/bin/env python
"""Clipping-error fixtures from the REAL reference (build container only):

  1. `-sm collect` on the seeded ResNet-18 of make_stats_golden.py (2 batches of 2 images, 64x64, int4), once per tensor
     and once with -pcq_a -baa, with the error columns filled -> the reference's summary files, copied to
     tests/golden/ref_stats_err/ (CSV + pickle);
  2. `-c mix -sm use` W4A4 on those files, per tensor and with -pcq_a -baa -> logits, and the per-layer (per-channel)
     choice the reference's rule makes from the collected mse columns, in tests/golden/ref_stats_err_logits.npz.

The reference never hands quantized tensors to save_tensor_stats.  In this process only, save_tensor_stats is wrapped so
that it receives tensors_q = {orig, lowp, gaus, laplace}: the outputs of the reference's own
gemmlowpClippingQuantize(tensor, id, tag, stat_id=None, clip_type=k) of the quantizer quantize_instant picks for that call
site in use mode (tag, 8-bit ignore list, half_range), with get_alpha returning (max - min) / 2 for 'lowp' (the alpha
get_alpha(clip_type='mix') computes for it).  The per-channel manager is built with collect_err=True.  The reference's
own formulas then write the columns.
"""
import functools
import os
import shutil
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_stats_golden as msg  # noqa: E402  (reference import, stubs, CPU leaf, scratch statistics directory)

from pytorch_quantizer.quantization.qtypes.int_quantizer import IntQuantizer  # noqa: E402

mc, iqm, sm_mod, smp_mod = msg.mc, msg.mc.iqm, msg.sm_mod, msg.smp_mod
OUT = os.path.join(HERE, "ref_stats_err")
HALF = {}   # activation id -> hasattr(module, 'before_relu')

_get_alpha = IntQuantizer.get_alpha


def get_alpha(self, tensor, tag="", stat_id=None, clip_type="laplace", per_channel=False):
    if clip_type == "lowp":
        stats = self.__act_stats_perchannel__ if per_channel else self.__act_stats__
        st = stats(tensor, ["min", "max"], avg_over_batch=False)
        return (st["max"] - st["min"]) / 2
    return _get_alpha(self, tensor, tag, stat_id, clip_type, per_channel)


IntQuantizer.get_alpha = get_alpha


def candidates(tensor, tag, id):
    """tensors_q of one call site: the use-mode quantizer of quantize_instant (inference_quantization_manager.py:549-562)."""
    if id.startswith("conv"):
        qtag, half = ("activation_classifier" if tensor.shape[1] == 1000 else "activation"), HALF[id]
    elif id.startswith("linear"):
        qtag, half = tag, (HALF[id] if "classifier" not in tag else False)
    elif id.startswith("maxpool"):
        qtag, half = "activation_pooling", False
    elif id.startswith("avgpool"):
        qtag, half = "", False
    else:  # bn: quantize_instant(out, "activation", ...) -> tag "" -> the default quantizer
        qtag, half = "", HALF[id]
    om = iqm.QMI().op_manager
    q = om.get_quantizer("ignored" if id in om.ignore_ids else qtag)
    q.half_range = half
    res = {"orig": tensor}
    for k in ("lowp", "gaus", "laplace"):
        res[k] = q.gemmlowpClippingQuantize(tensor, id, tag, stat_id=None, clip_type=k)
    return res


def wrap_save(cls, per_channel):
    orig = cls.save_tensor_stats

    def save(self, tensor, tag, id, tensors_q={}, force_global_min_max=False):
        skipped = per_channel and (len(tensor.shape) < 3 or (tensor.shape[2] == 1 and tensor.shape[3] == 1))
        tq = {} if skipped else candidates(tensor, tag, id)
        return orig(self, tensor, tag, id, tensors_q=tq, force_global_min_max=force_global_min_max)

    cls.save_tensor_stats = save


wrap_save(sm_mod.StatisticManager, False)
wrap_save(smp_mod.StatisticManagerPerChannel, True)
_pc_init = smp_mod.StatisticManagerPerChannel.__init__


@functools.wraps(_pc_init)
def _pc_init_err(self, folder, load_stats, *a, **k):
    k["collect_err"] = True
    _pc_init(self, folder, load_stats, *a, **k)


smp_mod.StatisticManagerPerChannel.__init__ = _pc_init_err


def run(flags, xs):
    """make_stats_golden.run, recording which call sites sit before a ReLU."""
    mc.Singleton._instances.clear()
    from itertools import count
    for cls in (iqm.Conv2dWithId, iqm.LinearWithId, iqm.MaxPool2dWithId, iqm.AvgPool2dWithId, iqm.BatchNorm2dWithId):
        cls._id = count(0)
    args = mc.make_args(arch="resnet18", stats_folder="resnet18", **flags)
    outs = []
    with iqm.QuantizationManagerInference(args, mc.qparams(args)) as qm:
        torch.manual_seed(12345)
        model = mc.models.resnet18(weights=None)
        mc.set_node_names(model)
        mc.resnet_mark_before_relu(model)
        mc.search_absorbe_bn(model)
        qm.bn_folding = True
        model.eval()
        for m in model.modules():
            for cls, fmt in ((iqm.Conv2dWithId, "conv%d_activation"), (iqm.LinearWithId, "linear%d_activation"),
                             (iqm.BatchNorm2dWithId, "bn%d_activation")):
                if isinstance(m, cls):
                    HALF[fmt % m.id] = hasattr(m, "before_relu")
        qm.quantize_model(model)
        with torch.no_grad():
            for x in xs:
                outs.append(model(x).numpy())
    return np.stack(outs)


def mix_choice(lowp, gaus, laplace):
    """int_quantizer.py:322-323 as an index into (lowp, gaus, laplace)."""
    c = np.where(np.asarray(gaus) < np.asarray(laplace), 1, 2)
    return np.where(np.asarray(lowp) < np.asarray(gaus), 0, c)


W4A4 = dict(qtype="int4", qweight="int4", clipping="mix", per_channel_quant_weights=True, bit_alloc_weight=True,
            bias_corr_weight=True)
PCQ = dict(per_channel_quant_act=True, bit_alloc_act=True)


def main():
    import pickle
    import pandas as pd
    torch.set_num_threads(8)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    xs = msg.batches()
    run(dict(stats_mode="collect", qtype="int4", qweight="int4"), xs)
    run(dict(stats_mode="collect", qtype="int4", qweight="int4", **PCQ), xs)
    out = {"use_mix_w4a4": run(dict(stats_mode="use", **W4A4), xs),
           "use_mix_w4a4_pcq": run(dict(stats_mode="use", **W4A4, **PCQ), xs)}
    csv = os.path.join(msg.SCRATCH, "statistics", "resnet18", "resnet18_summary.csv")
    pkl = os.path.join(msg.SCRATCH, "statistics", "per_channel", "resnet18", "resnet18_statistics_perchannel_summary.pkl")
    df = pd.read_csv(csv, index_col=0)
    for layer in df.index:
        out["choice_tensor/" + layer] = mix_choice(*(df.loc[layer, "mean_mse_" + k] for k in ("lowp", "gaus", "laplace")))
    with open(pkl, "rb") as f:
        pc = pickle.load(f)
    for layer, frame in pc.items():
        out["choice_channel/" + layer] = mix_choice(*(frame["mean_mse_" + k].to_numpy() for k in ("lowp", "gaus", "laplace")))
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(os.path.join(OUT, "statistics", "resnet18"))
    os.makedirs(os.path.join(OUT, "statistics", "per_channel", "resnet18"))
    shutil.copy(csv, os.path.join(OUT, "statistics", "resnet18"))
    shutil.copy(pkl, os.path.join(OUT, "statistics", "per_channel", "resnet18"))
    np.savez_compressed(os.path.join(HERE, "ref_stats_err_logits.npz"), **out)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    for k, v in out.items():
        if k.startswith("use"):
            print(k, v.shape, float(np.abs(v).mean()))
    print(df[[c for c in df.columns if c.startswith("mean_mse") or c.startswith("mean_cos")]].head(8))


if __name__ == "__main__":
    main()
