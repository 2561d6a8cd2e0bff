#!/usr/bin/env python
"""Use-mode (`-sm use`) launch parameters of ``IntQuantizer``, written to use_params.npz.

Every case builds a quantizer, attaches fake statistics (and, for `-c mse` / `-bap mse`, fake curves and tables), calls
it twice on the same call site with ``ops.quantize1``, ``quantize1_bca``, ``float2gemmlowp`` and ``fused`` replaced by
recorders, and keeps the values each launch got: delta, offset, bits, num_bits and layout of the torch leaf; range,
offset and preserve_zero of the compiled leaf; the sum of the tensor the leaf was handed and whether it is the caller's.  A case the quantizer refuses keeps the
exception's type.  tests/test_use_params_cpu.py runs the same cases and compares bit for bit; it also checks that the
second call reads no statistics.

    python tests/golden/make_use_params_golden.py
"""
import contextlib
import itertools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "use_params.npz")

C = 4
RULES = ["no", "laplace", "gaus", "2.5std", "mix", "mse", "kld"]
PRIORS = [None, "gaus", "laplace", "mse"]   # -baa off, or -baa -bap <prior>


def _stats(per_channel):
    """{kind_stat: value}: float32 [C] vectors per channel, float64 scalars per tensor (what the summary files give)."""
    rs = np.random.RandomState(7)
    out = {}
    for kind, shift in (("mean", 0.0), ("min", -0.5), ("max", 0.5)):
        v = {"min": -rs.rand(C) * 2 - 0.1 + shift, "max": rs.rand(C) * 3 + 0.2 + shift, "mean": rs.randn(C) * 0.2,
             "b": rs.rand(C) + 0.2, "std": rs.rand(C) * 1.5 + 0.3, "kld_th": rs.rand(C) * 2 + 0.5,
             "mse_lowp": np.array([3.0, 0.5, 1.0, 2.0]), "mse_gaus": np.array([1.0, 1.0, 1.0, 2.5]),
             "mse_laplace": np.array([2.0, 0.1, 1.0, 1.5])}
        for k, a in v.items():
            out["%s_%s" % (kind, k)] = a.astype(np.float32) if per_channel else np.float64(a[1])
    return out


class Reads(object):
    def __init__(self):
        self.n = 0


class FakeStats(object):
    def __init__(self, per_channel, reads):
        self.table, self.reads = _stats(per_channel), reads

    def get_tensor_stat(self, id, stat, kind="mean"):
        self.reads.n += 1
        return self.table["%s_%s" % (kind, stat)]


class FakeCurves(object):
    """ClipMseStatistics.best: m* per group and the prior of the curve."""

    def __init__(self, per_channel, reads):
        self.m = np.float32([1.5, 4.0, 2.5, 8.0]) if per_channel else np.float32([3.0])
        self.prior, self.reads = ("laplace" if per_channel else "gaus"), reads

    def best(self, id):
        self.reads.n += 1
        return self.m, self.prior


class FakeTables(object):
    """BitMseStatistics.table / multipliers_of: per-channel errors of widths 0..8 measured under ``rule``."""

    def __init__(self, rule, reads):
        scale = np.array([4.0, 0.25, 1e-6, 1.0])
        self.mse = scale[:, None] * 4.0 ** -np.arange(9)[None, :]
        self.m = (1.0 + 0.5 * np.arange(9)[None, :] + np.arange(C)[:, None]).astype(np.float32)
        self.rule, self.reads = rule, reads

    def table(self, id):
        self.reads.n += 1
        return self.mse, self.rule

    def multipliers_of(self, id):
        self.reads.n += 1
        return self.m, "laplace"


def _np(v):
    if v is None:
        return None
    return v.detach().cpu().numpy().copy() if isinstance(v, torch.Tensor) else np.asarray(v)


class Recorder(object):
    """ops.quantize1 / quantize1_bca / float2gemmlowp / fused with the values they were handed."""

    def __init__(self):
        self.calls = []
        self.input = None   # the tensor handed to the quantizer

    def _add(self, entry, x, out, **vals):
        rec = {"entry": np.asarray(entry), "x_sum": np.float64(x.double().sum()), "x_is_input": np.asarray(x is self.input),
               "out": np.asarray(out is not None)}
        rec.update({k: _np(v) for k, v in vals.items() if v is not None})
        self.calls.append(rec)

    def quantize1(self, x, delta, offset, num_bits, bits=None, layout=None, want_grid=False, out=None, bias=None):
        self._add("quantize1", x, out, delta=delta, offset=offset, num_bits=num_bits, bits=bits, layout=layout, bias=bias)
        return out if out is not None else torch.zeros_like(x)

    def quantize1_bca(self, x, delta, offset, num_bits, bits=None, bias=None, relu_first=False, out=None, want_qbias=False):
        self._add("quantize1_bca", x, out, delta=delta, offset=offset, num_bits=num_bits, bits=bits, bias=bias,
                  relu_first=relu_first)
        return out if out is not None else torch.zeros_like(x)

    def float2gemmlowp(self, x, range_, offset, num_bits, int_exp, enforce_true_zero, noise=None, out=None):
        self._add("float2gemmlowp", x, out, range=range_, offset=offset, num_bits=num_bits, preserve_zero=enforce_true_zero)
        return out if out is not None else torch.zeros_like(x)

    def fused(self, x, layout, out=None, **kw):
        self._add("fused", x, out, layout=layout)
        return torch.zeros_like(x)


@contextlib.contextmanager
def recording():
    from cnn_quantization_b200 import ops
    rec = Recorder()
    saved = {k: getattr(ops, k) for k in ("quantize1", "quantize1_bca", "float2gemmlowp", "fused")}
    for k in saved:
        setattr(ops, k, getattr(rec, k))
    try:
        yield rec
    finally:
        for k, v in saved.items():
            setattr(ops, k, v)


def cases():
    """(name, settings) of the matrix: rule x per channel / per tensor x positive x -baa prior x int4 / int8 x stats_kind,
    with a convolution bias the kernel takes and the in-place activations of the manager; then the -bca fallback and
    the out-of-place bias on the per-tensor routes."""
    out = []
    for rule, pc, pos, prior, bits, kind in itertools.product(RULES, (True, False), (False, True), PRIORS, (4, 8),
                                                              ("mean", "max")):
        name = "%s-%s-%s-%s-int%d-%s" % (rule, "pc" if pc else "pt", "pos" if pos else "sgn", prior or "nobaa", bits, kind)
        out.append((name, dict(rule=rule, pc=pc, pos=pos, prior=prior, bits=bits, kind=kind, bca=None, inplace=True)))
    for rule, pos, bca in itertools.product(RULES, (False, True), (None, False, True)):
        name = "%s-pt-%s-bca%s-copy" % (rule, "pos" if pos else "sgn", {None: "off", False: "", True: "relu"}[bca])
        out.append((name, dict(rule=rule, pc=False, pos=pos, prior=None, bits=4, kind="mean", bca=bca, inplace=False)))
    return out


def run_case(s):
    """([record of each launch of the two calls], statistics reads after the first call, after the second), or the
    refusal's exception type name in place of the records."""
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    p = dict(clipping="no" if s["rule"] == "kld" else s["rule"], stats_kind=s["kind"], kld=s["rule"] == "kld",
             pcq_weights=False, pcq_act=s["pc"], bit_alloc_act=s["prior"] is not None, bit_alloc_weight=False,
             bcorr_act=s["bca"] is not None, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior=s["prior"] or "gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None,
             measure_entropy=False, logger=None, mtd_quant=False)
    q = IntQuantizer(s["bits"], p)
    reads = Reads()
    sm = FakeStats(s["pc"], reads)
    q.sm = lambda: sm
    q.mse_curves = FakeCurves(s["pc"], reads)
    q.bit_tables = FakeTables(q.clipping, reads)
    q.half_range = s["pos"]
    q.inplace = s["inplace"]
    g = torch.Generator().manual_seed(3)
    bias = torch.randn(C, generator=g)
    counts = []
    with recording() as rec:
        for _ in range(2):
            x = rec.input = torch.randn(2, C, 4, 4, generator=g)
            try:
                q(x, "conv1", "activation", stat_id="conv1_activation", bias=bias, bias_correct=s["bca"])
            except Exception as e:   # a refusal: the same on both calls
                rec.calls.append({"raise": np.asarray(type(e).__name__)})
            counts.append(reads.n)
    return rec.calls, counts


def pack(name, calls):
    """{"<name>::<launch>::<field>": (dtype and shape, or the string's value; float64 values)} of ``run_case``'s records."""
    out = {}
    for i, rec in enumerate(calls):
        for k, v in rec.items():
            if v.dtype.kind == "U":
                out["%s::%d::%s" % (name, i, k)] = ("str " + str(v), np.zeros(0))
            else:
                out["%s::%d::%s" % (name, i, k)] = ("%s%s" % (v.dtype, v.shape), v.astype(np.float64).reshape(-1))
    return out


def save(path, packed):
    keys = sorted(packed)
    np.savez_compressed(path, keys=np.array(keys), kinds=np.array([packed[k][0] for k in keys]),
                        sizes=np.array([packed[k][1].size for k in keys]),
                        values=np.concatenate([packed[k][1] for k in keys]))


def load(path):
    d = np.load(path)
    values = np.split(d["values"], np.cumsum(d["sizes"])[:-1])
    return {str(k): (str(kind), v) for k, kind, v in zip(d["keys"], d["kinds"], values)}


def main():
    packed = {}
    for name, s in cases():
        packed.update(pack(name, run_case(s)[0]))
    save(OUT, packed)
    print("wrote %d records of %d cases to %s" % (len(packed), len(cases()), OUT))


if __name__ == "__main__":
    main()
