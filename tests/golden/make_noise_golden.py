#!/usr/bin/env python
"""Quantization-noise fixtures (`-ms` with the reference's measure_statistics module) from the REAL reference (build
container only), written to ref_noise/*.npz:

  1. synthetic.npz: the reference's own ``MeasureStatistics.save_measure(y, y_with_noise, x, w, id)`` on seeded cases -
     4-D and 2-D tensors, a zero sample, y == y_with_noise, and a row whose |mean| / std is about 1e3 - with the inputs;
  2. <config>.npz: the unmodified reference manager on the seeded ResNet-18 of make_stats_golden.py (2 batches of 4
     images, 64x64) in three configurations.  The reference cannot run this module as it stands: its import is commented
     out (inference_quantization_manager.py:10-11), the manager constructs ``MS(args.arch)`` while the module's
     constructor takes no argument, and the call sites pass only the tensor they hand on.  So the manager's ``MS`` is
     rebound to a small adapter (as make_angle_golden.py rebinds it to angle_stats) that feeds the module's own
     ``save_measure`` what it asks for: y and y_with_noise captured around ``quantize_instant`` (y itself where nothing
     is quantized), and the input and weight of the conv / linear being run.  The module writes <id>.csv itself; each
     config's files become one array per id (``ids`` in call order).

The compiled leaf runs on the CPU restatement, as in make_census.py.
"""
import os
import shutil
import sys

import numpy as np
import pandas as pd
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_stats_golden as msg  # noqa: E402  (reference import, stubs, CPU leaf, scratch statistics directory)

from pytorch_quantizer.quantization.inference import measure_statistics as ns_mod  # noqa: E402

OUT = os.path.join(HERE, "ref_noise")
CONFIGS = {
    "w4a4": dict(msg.W4A4),
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
}
_seen = {}   # what the running conv / linear handed the quantizer and got back, its input and weight


class _Adapter(object):
    """``MS(arch)`` of the reference manager: the module's MeasureStatistics with the missing arguments filled in."""

    def __init__(self, arch):
        self.ms = ns_mod.MeasureStatistics()
        self.ms.folder, self.ms.subfolder = os.path.join(msg.SCRATCH, "noise"), arch
        _seen["adapter"] = self

    @property
    def enabled(self):
        return self.ms.enabled

    def save_measure(self, out, id):
        y = _seen.pop("y", out)
        self.ms.save_measure(y, out, _seen["x"], _seen["w"], id)

    def __enter__(self):
        self.ms.__enter__()
        return self

    def __exit__(self, *args):
        self.ms.__exit__(*args)


def _install():
    iqm = msg.mc.iqm
    iqm.MS = _Adapter
    orig_q = iqm.TruncationOpManagerInference.quantize_instant

    def quantize_instant(self, tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False):
        y = tensor.clone()
        res = orig_q(self, tensor, id, tag, stat_id, half_range, override_att, verbose)
        _seen["y"] = y
        return res

    iqm.TruncationOpManagerInference.quantize_instant = quantize_instant
    for cls in (iqm.Conv2dWithId, iqm.LinearWithId):
        def forward(self, input, __orig=cls.forward):
            _seen.pop("y", None)
            _seen["x"], _seen["w"] = input, self.weight.detach()
            return __orig(self, input)

        cls.forward = forward


def batches():
    rs = np.random.RandomState(2026)
    return [torch.from_numpy(rs.standard_normal((4, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def synthetic_cases():
    g = torch.Generator().manual_seed(7)
    rnd = lambda *s: torch.randn(*s, generator=g)
    cases = {}
    y = rnd(4, 3, 5, 5)
    y[1] = 0.
    yq = torch.round(y * 8) / 8
    cases["conv4d"] = (y, yq, torch.relu(rnd(4, 2, 7, 7)), rnd(3, 2, 3, 3))
    y = rnd(5, 10)
    cases["linear2d"] = (y, torch.round(y * 4) / 4, rnd(5, 20), rnd(10, 20))
    y = rnd(3, 2, 4, 4)
    cases["identical"] = (y, y.clone(), rnd(3, 6, 4, 4), rnd(2, 6, 1, 1))
    y = 1000. + rnd(3, 64)
    y[1] = -1000. + y[1] - 1000.
    cases["large_mean"] = (y, torch.round(y * 4) / 4, 500. + rnd(3, 32), 3. + rnd(64, 32) * 3e-3)
    return cases


def main():
    torch.set_num_threads(8)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    arrays = {}
    for name, (y, yq, x, w) in synthetic_cases().items():
        ms = ns_mod.MeasureStatistics()
        ms.__enter__()
        ms.save_measure(y, yq, x, w, name)
        arrays.update({name + "_y": y.numpy(), name + "_yq": yq.numpy(), name + "_x": x.numpy(), name + "_w": w.numpy(),
                       name + "_ref": ms.stats[name]})
        msg.mc.Singleton._instances.clear()
    np.savez_compressed(os.path.join(OUT, "synthetic.npz"), columns=np.array(ns_mod.MeasureStatistics().stats_names),
                        **arrays)
    msg.mc.Singleton._instances.clear()
    _install()
    xs = batches()
    for name, flags in CONFIGS.items():
        msg.run(dict(measure_stats=True, **flags), xs)
        folder = os.path.join(msg.SCRATCH, "noise", "resnet18")
        ids = list(_seen["adapter"].ms.stats)   # call order
        assert sorted(ids) == sorted(f[:-4] for f in os.listdir(folder))
        frames = {i: pd.read_csv(os.path.join(folder, i + ".csv"), float_precision="round_trip") for i in ids}
        cols = list(frames[ids[0]].columns)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), ids=np.array(ids), columns=np.array(cols),
                            **{"id%03d" % k: frames[i].to_numpy(dtype=np.float64) for k, i in enumerate(ids)})
        print(name, len(ids), frames[ids[0]].shape, ids[:3], "...")
        shutil.rmtree(os.path.join(msg.SCRATCH, "noise"), ignore_errors=True)
    shutil.rmtree(msg.SCRATCH, ignore_errors=True)


if __name__ == "__main__":
    main()
