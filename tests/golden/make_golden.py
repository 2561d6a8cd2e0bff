#!/usr/bin/env python
"""Generate the CPU golden fixtures by running the REAL reference (read-only, at REF below).

Run only where the reference is checked out (no GPU needed):

    python tests/golden/make_golden.py            # writes tests/golden/ref_cpu_*.npz + ref_census.json

The reference has no tests or golden vectors of its own (SURVEY.md section 4), so the fixtures are the
reference's *outputs*: its pure-PyTorch hot path (int_quantizer.py) executed on CPU tensors with a
stub `int_quantization` module (the compiled leaf needs a GPU: it is compared live with the reference's own extension
on the GPU, tests/test_gpu_ref_ext.py and tests/test_gpu_ref_live.py).  Inputs are drawn from numpy RandomState (stable across versions) and stored
in the fixture next to the outputs.  Nothing here is imported by the product or by the GPU tests.
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from golden_inputs import regen  # noqa: E402
REF = "/root/reference"


def _import_reference():
    sys.path.insert(0, REF)
    stub = types.ModuleType("int_quantization")

    def _no_gpu(*a, **k):
        raise RuntimeError("compiled leaf needs a GPU")

    stub.float2gemmlowp = _no_gpu
    sys.modules["int_quantization"] = stub
    import pytorch_quantizer.quantization.qtypes.int_quantizer  # noqa: F401  (the package re-exports a function of the same name)
    return sys.modules["pytorch_quantizer.quantization.qtypes.int_quantizer"]


def base_params(**over):
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=False,
             bit_alloc_act=False, bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False,
             vcorr_weight=False, bit_alloc_rmode="round", bit_alloc_prior="gaus",
             bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p.update(over)
    return p


def main():
    iq = _import_reference()
    IntQuantizer = iq.IntQuantizer
    out = {}
    meta = {}

    # capture what the leaf receives (delta, offset, bit_alloc) for the stats-driven cases
    captured = {}
    orig_leaf = IntQuantizer.__gemmlowpQuantize1__

    def spy(self, tensor, delta, offset, bit_alloc=None, measure_entropy=False):
        captured["delta"] = torch.as_tensor(delta, dtype=torch.float32).detach().clone()
        captured["offset"] = torch.as_tensor(offset, dtype=torch.float32).detach().clone()
        captured["bits"] = None if bit_alloc is None else bit_alloc.detach().clone()
        return orig_leaf(self, tensor, delta, offset, bit_alloc, measure_entropy)

    IntQuantizer.__gemmlowpQuantize1__ = spy

    # Device-semantics shim.  get_alpha_mult (int_quantizer.py:139-141) does `omega = omega.cpu().numpy()` and
    # then `omega *= 2` for one-sided ranges.  On the CUDA tensors the reference is written for, `.cpu()` is a
    # copy; on CPU tensors it aliases and the caller's omega is doubled as a side effect - an artefact of running
    # the reference on CPU, not part of its algorithm.  Hand it a clone so the fixtures carry the CUDA behaviour.
    orig_mult = IntQuantizer.get_alpha_mult
    IntQuantizer.get_alpha_mult = staticmethod(lambda omega, sym=True: orig_mult(omega.clone(), sym=sym))

    def add(name, x, y, info):
        # inputs are regenerated from info["input"] by tests/golden/golden_inputs.py (numpy RandomState)
        assert np.array_equal(x, regen(info["input"])), name
        out[name + ".y"] = y.detach().numpy() if isinstance(y, torch.Tensor) else y
        for k in ("delta", "offset", "bits"):
            v = captured.get(k)
            if v is not None:
                out[name + "." + k] = v.numpy().reshape(-1)
        meta[name] = info
        captured.clear()

    # ---- a3: leaf with given parameters --------------------------------------------------
    # config 1 of BASELINE.json: int4 per-tensor on 1x64x56x56, params = global min/max
    spec = dict(seed=12345, shape=(1, 64, 56, 56), chan_scale=False)
    x = regen(spec)
    q = iq.int_quantizer("int4", base_params())
    xt = torch.from_numpy(x)
    y = q.__gemmlowpQuantize1__(xt, xt.max() - xt.min(), xt.min())
    add("leaf_cfg1_int4", x, y, dict(kind="leaf", num_bits=4, input=spec))

    for bits in (2, 8):
        spec = dict(seed=100 + bits, shape=(3, 5, 6, 7), chan_scale=False)
        x = regen(spec)
        q = iq.int_quantizer("int%d" % bits, base_params())
        xt = torch.from_numpy(x)
        y = q.__gemmlowpQuantize1__(xt, xt.max() - xt.min(), xt.min())
        add("leaf_tensor_int%d" % bits, x, y, dict(kind="leaf", num_bits=bits, input=spec))

    # per-row parameters with per-row bit widths (0..8), incl. qmax==0 rows and a degenerate row
    spec = dict(seed=7, shape=(12, 333), const_row=(5, 0.75))  # constant row: delta == 0 -> scale floor 1e-8
    x = regen(spec)
    xt = torch.from_numpy(x)
    mn, mx = xt.min(-1)[0], xt.max(-1)[0]
    bits = torch.tensor([0, 1, 2, 3, 4, 5, 6, 7, 8, 4, 0, 3], dtype=torch.float32)
    q = iq.int_quantizer("int4", base_params())
    y = q.__gemmlowpQuantize1__(xt, mx - mn, mn, bit_alloc=bits)
    add("leaf_rows_bits", x, y, dict(kind="leaf_rows", num_bits=4, input=spec))
    y = q.__gemmlowpQuantize1__(xt, mx - mn, mn)
    add("leaf_rows_nobits", x, y, dict(kind="leaf_rows", num_bits=4, input=spec))

    # ---- a6/a4/a7/a8/a9/a10: activation paths, on-the-fly statistics ---------------------
    act_cases = [
        # name, shape, bits, params, half_range, relu
        ("act_lap_tensor_cfg1", (1, 64, 56, 56), 4, dict(clipping="laplace"), False, False),
        ("act_lap_tensor_cfg1_hr", (1, 64, 56, 56), 4, dict(clipping="laplace"), True, True),
        ("act_lap_tensor_2d", (16, 200), 4, dict(clipping="laplace", pcq_act=True), False, False),
        ("act_lap_pc", (4, 16, 14, 14), 4, dict(clipping="laplace", pcq_act=True), False, False),
        ("act_lap_pc_hr", (4, 16, 14, 14), 4, dict(clipping="laplace", pcq_act=True), True, False),
        ("act_lap_pc_ba", (4, 16, 14, 14), 4, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), False, False),
        ("act_lap_pc_ba_hr", (4, 16, 14, 14), 4, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), True, False),
        ("act_lap_pc_ba_hr_relu", (6, 24, 7, 7), 4, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), True, True),
        ("act_lap_pc_ba_odd", (5, 12, 7, 7), 4, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), False, False),
        ("act_lap_pc_ba_lapprior", (4, 16, 14, 14), 4,
         dict(clipping="laplace", pcq_act=True, bit_alloc_act=True, bit_alloc_prior="laplace"), False, False),
        ("act_lap_pc_ba_ceil", (4, 16, 14, 14), 4,
         dict(clipping="laplace", pcq_act=True, bit_alloc_act=True, bit_alloc_rmode="ceil"), False, False),
        ("act_lap_pc_ba_t53", (4, 32, 8, 8), 4,
         dict(clipping="laplace", pcq_act=True, bit_alloc_act=True, bit_alloc_target_act=5.3), True, True),
        ("act_lap_pc_ba_int3", (3, 20, 9, 5), 3, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), False, False),
        ("act_lap_pc_int8_noba", (3, 10, 6, 6), 8, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), False, False),
        ("act_gaus_pc", (4, 16, 14, 14), 4, dict(clipping="gaus", pcq_act=True), False, False),
        ("act_gaus_tensor_hr", (4, 16, 14, 14), 4, dict(clipping="gaus"), True, True),
        ("act_2std_pc", (4, 16, 14, 14), 4, dict(clipping="2std", pcq_act=True), False, False),
        ("act_pc_noclip", (4, 16, 14, 14), 4, dict(pcq_act=True), False, False),
        ("act_pc_noclip_hr", (4, 16, 14, 14), 4, dict(pcq_act=True), True, True),
        ("act_pc_noclip_ba", (4, 16, 14, 14), 4, dict(pcq_act=True, bit_alloc_act=True), False, False),
        ("act_pc_noclip_ba_lap", (4, 16, 14, 14), 4, dict(pcq_act=True, bit_alloc_act=True, bit_alloc_prior="laplace"), True, True),
    ]
    for i, (name, shape, bits, over, hr, relu) in enumerate(act_cases):
        spec = dict(seed=1000 + i, shape=shape, dist="laplace" if i % 2 else "normal", relu=relu)
        x = regen(spec)
        q = iq.int_quantizer("int%d" % bits, base_params(**over))
        q.pcq_w = False  # as the manager does for activation quantizers (inference_quantization_manager.py:455-458)
        q.half_range = hr
        y = q(torch.from_numpy(x), "conv1_activation", "activation")
        add(name, x, y, dict(kind="act", num_bits=bits, params=over, half_range=hr, input=spec))

    # force_positive (fused-relu archs) is handled exactly like half_range
    spec = dict(seed=77, shape=(4, 16, 14, 14), relu=True)
    x = regen(spec)
    q = iq.int_quantizer("int4", base_params(clipping="laplace", pcq_act=True, bit_alloc_act=True))
    q.pcq_w = False
    q.force_positive = True
    y = q(torch.from_numpy(x), "conv1_activation", "activation")
    add("act_lap_pc_ba_forcepos", x, y, dict(kind="act", num_bits=4,
                                             params=dict(clipping="laplace", pcq_act=True, bit_alloc_act=True),
                                             half_range=False, force_positive=True, input=spec))

    # ---- a5: weights per output channel ---------------------------------------------------
    w_cases = [
        ("w_pc_int4", (16, 8, 3, 3), 4, dict(pcq_weights=True)),
        ("w_pc_int4_ba", (16, 8, 3, 3), 4, dict(pcq_weights=True, bit_alloc_weight=True)),
        ("w_pc_int4_ba_t53", (32, 4, 3, 3), 4, dict(pcq_weights=True, bit_alloc_weight=True, bit_alloc_target_weight=5.3)),
        ("w_pc_int8_fc", (10, 64), 8, dict(pcq_weights=True, bit_alloc_weight=True)),
        ("w_pc_int4_first", (8, 3, 7, 7), 4, dict(pcq_weights=True, bit_alloc_weight=True)),  # override num_bits=8
    ]
    for i, (name, shape, bits, over) in enumerate(w_cases):
        spec = dict(seed=2000 + i, shape=shape, mult=0.05)
        x = regen(spec)
        q = iq.int_quantizer("int%d" % bits, base_params(**over))
        q.pcq_a = False
        q.clipping = "no"
        ov = ("num_bits", 8) if name.endswith("first") else None
        y = q(torch.from_numpy(x), "w", "weight", override_att=ov)
        add(name, x, y, dict(kind="weight", num_bits=bits, params=over, override_num_bits=8 if ov else None, input=spec))

    # ---- a12: mid-tread ----------------------------------------------------------------------
    mt_cases = [
        ("mt_act_pc_sym", (4, 16, 14, 14), dict(clipping="laplace", pcq_act=True, mtd_quant=True, bit_alloc_target_act=5.3), False, False),
        ("mt_act_pc_pos", (4, 16, 14, 14), dict(clipping="laplace", pcq_act=True, mtd_quant=True, bit_alloc_target_act=5.3), True, True),
        ("mt_act_tensor", (8, 300), dict(clipping="laplace", pcq_act=True, mtd_quant=True, bit_alloc_target_act=4.0), False, False),
        ("mt_act_pc_t4", (3, 10, 6, 6), dict(clipping="laplace", pcq_act=True, mtd_quant=True), False, False),
    ]
    for i, (name, shape, over, hr, relu) in enumerate(mt_cases):
        spec = dict(seed=3000 + i, shape=shape, dist="laplace", relu=relu)
        x = regen(spec)
        q = iq.int_quantizer("int4", base_params(**over))
        q.pcq_w = False
        q.half_range = hr
        y = q(torch.from_numpy(x), "conv1_activation", "activation")
        add(name, x, y, dict(kind="act", num_bits=4, params=over, half_range=hr, input=spec))
    spec = dict(seed=3100, shape=(16, 8, 3, 3), mult=0.05)
    x = regen(spec)
    q = iq.int_quantizer("int4", base_params(pcq_weights=True, mtd_quant=True, bit_alloc_target_weight=5.3))
    q.pcq_a = False
    q.clipping = "no"
    y = q(torch.from_numpy(x), "w", "weight")
    add("mt_w_pc", x, y, dict(kind="weight", num_bits=4,
                              params=dict(pcq_weights=True, mtd_quant=True, bit_alloc_target_weight=5.3), input=spec))

    # ---- a9 known answers + tables ------------------------------------------------------------
    rs = np.random.RandomState(99)
    sig = rs.uniform(0.05, 4.0, size=256).astype(np.float32)
    out["bits.sigma"] = sig
    for tgt, rmode in ((4, True), (4, False), (5.3, True), (3, True), (2, True)):
        b = IntQuantizer.get_bits_alloc_fixed_target(torch.from_numpy(sig), tgt, rmode)
        out["bits.t%s_%s" % (str(tgt).replace(".", "p"), "round" if rmode else "ceil")] = b.numpy()
    out["tables.omega"] = iq.omega_table
    out["tables.alpha"] = iq.alpha_table
    om = torch.tensor([0.3, 1.0, 2.0, 3.7, 16.0, 40.5, 256.0, 900.0])
    out["tables.mult_in"] = om.numpy()
    out["tables.mult_sym"] = IntQuantizer.get_alpha_mult(om.clone(), sym=True)
    out["tables.mult_pos"] = IntQuantizer.get_alpha_mult(om.clone()[:6], sym=False)

    # ---- a10 statistics -------------------------------------------------------------------------
    x = regen(dict(seed=4000, shape=(6, 10, 5, 7)))
    xt = torch.from_numpy(x)
    names = ["min", "max", "mean", "b", "std"]
    for k, v in IntQuantizer.__act_stats__(xt, names, avg_over_batch=False).items():
        out["stats.tensor." + k] = v.numpy().reshape(-1)
    for k, v in IntQuantizer.__act_stats__(xt, names, avg_over_batch=True).items():
        out["stats.sampleavg." + k] = v.numpy().reshape(-1)
    for k, v in IntQuantizer.__act_stats_perchannel__(xt, names, avg_over_batch=False).items():
        out["stats.pc." + k] = v.numpy()
    for k, v in IntQuantizer.__act_stats_perchannel__(xt, names, avg_over_batch=True).items():
        out["stats.pcavg." + k] = v.numpy()

    IntQuantizer.__gemmlowpQuantize1__ = orig_leaf
    np.savez_compressed(os.path.join(HERE, "ref_cpu.npz"), **out)
    with open(os.path.join(HERE, "ref_cpu_meta.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    print("wrote", len(out), "arrays,", len(meta), "cases")


if __name__ == "__main__":
    torch.set_num_threads(1)
    main()
