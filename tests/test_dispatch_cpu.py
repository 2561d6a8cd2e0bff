"""Which launch ``IntQuantizer.__call__`` chooses, with which fusion arguments, and how it tags the result.

``ops.fused``, ``ops.quantize1``, ``ops.quantize1_bca`` and ``ops.float2gemmlowp`` are replaced by recorders that return
CPU tensors of the right shape, so the dispatch runs without a GPU.  The layout predicates the dispatch consults are the
real ones, and the cases sit on their boundaries: channel counts around 4 / 896 / 2048, batch sizes around 4096, odd and
too small H / W, NCHW against channels-last memory, a view at storage offset 1, residuals with other strides or dtype, and
deferred shortcuts with a matching or a different bias.

A recorded call reads ``"<entry point> <flag> ..."`` (flags in any order):
``cl`` channels_last, ``any`` any_dense_format, ``given`` range_mode == RANGE_GIVEN, ``stats`` stats_only, ``out`` an
output tensor, ``bias``, ``bp<n>`` bias_period, ``res`` / ``rstats`` / ``rbias`` residual / residual_stats /
residual_bias, ``hist``, ``pool2`` / ``pool3``; for quantize1: ``layout``; for quantize1_bca: ``relu`` (relu_first).
Result tags: ``nonneg`` (_fq_nonneg current), ``res`` (_fq_residual_fused), ``defer`` (_fq_deferred, carrying the bias
the call got), ``pool2`` / ``pool3`` (_fq_pooled)."""
import numpy as np
import pytest
import torch

from cnn_quantization_b200 import _lib as L, ops
from cnn_quantization_b200.int_quantizer import IntQuantizer

BASE = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=False, bit_alloc_act=False,
            bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
            bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
            logger=None, mtd_quant=False)

QUANT = {
    # per-channel ACIQ Laplace with bit allocation (W4A4 activations)
    "pc": (4, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True)),
    "pc_me": (4, dict(clipping="laplace", pcq_act=True, bit_alloc_act=True, measure_entropy=True)),
    # per-channel min / max
    "pcmm": (4, dict(pcq_act=True)),
    # per-sample / per-tensor min / max, compiled leaf (int8: the rows kernel)
    "int8": (8, dict()),
    "int8_me": (8, dict(measure_entropy=True)),
    # per-channel mid-tread
    "mtd": (4, dict(clipping="laplace", pcq_act=True, mtd_quant=True)),
    "mtd_me": (4, dict(clipping="laplace", pcq_act=True, mtd_quant=True, measure_entropy=True)),
    # per-tensor ACIQ Laplace
    "pt": (4, dict(clipping="laplace")),
}


class Recorder(object):
    def __init__(self):
        self.calls = []

    def _add(self, name, **flags):
        self.calls.append(" ".join([name] + sorted(k for k, on in flags.items() if on)))

    def fused(self, x, layout, *, out=None, stats_only=False, want_stats=False, pool=None, bias_period=0, **kw):
        flags = dict(cl=kw.get("channels_last"), any=kw.get("any_dense_format"), given=kw.get("range_mode") == L.RANGE_GIVEN,
                     stats=stats_only, out=out is not None, bias=kw.get("bias") is not None,
                     res=kw.get("residual") is not None, rstats=kw.get("residual_stats") is not None,
                     rbias=kw.get("residual_bias") is not None, hist=kw.get("hist") is not None)
        flags["bp%d" % bias_period] = bias_period != 0
        if pool is not None:
            assert tuple(pool) in ((2, 2), (3, 3))
            flags["pool%d" % pool[0]] = True
        self._add("fused", **flags)
        stats = torch.zeros((int(layout[1]), L.STATS_STRIDE))
        if stats_only:
            return stats
        if pool is not None:
            n, c, h, w = x.shape
            res = torch.zeros((n, c, h // 2, w // 2)).contiguous(memory_format=torch.channels_last)
        else:
            res = out if out is not None else torch.zeros_like(x)
        return (res, stats) if want_stats else res

    def quantize1(self, x, delta, offset, num_bits, bits=None, layout=None, want_grid=False, out=None, bias=None):
        self._add("quantize1", layout=layout is not None, out=out is not None, bias=bias is not None)
        return out if out is not None else torch.zeros_like(x)

    def quantize1_bca(self, x, delta, offset, num_bits, bits=None, bias=None, relu_first=False, out=None, want_qbias=False):
        self._add("bca", relu=relu_first, out=out is not None, bias=bias is not None)
        return out if out is not None else torch.zeros_like(x)

    def float2gemmlowp(self, x, range_, offset, num_bits, int_exp, enforce_true_zero, noise=None, out=None):
        self._add("float2gemmlowp", out=out is not None)
        return out if out is not None else torch.zeros_like(x)


class FakeStats(object):
    """``-sm use`` statistics: C-element vectors for per-channel quantizers, scalars otherwise."""

    def __init__(self, c):
        self.c = c

    def get_tensor_stat(self, id, stat, kind):
        v = {"min": -1.0, "max": 2.0, "mean": 0.25, "b": 0.5, "std": 0.7}[stat]
        if self.c is None:
            return v
        return (v * (1.0 + 0.01 * np.arange(self.c))).astype(np.float32)


def _tensor(shape, fmt, seed=0):
    """``fmt``: "nchw", "cl" (channels-last), "mis" (channels-last strides at storage offset 1: 4-byte aligned only)."""
    g = torch.Generator().manual_seed(seed)
    if fmt == "mis":
        n, c, h, w = shape
        x = torch.randn(n * c * h * w + 1, generator=g)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
        assert x.data_ptr() % 16 != 0
        return x
    x = torch.randn(shape, generator=g)
    x = x.contiguous(memory_format=torch.channels_last) if fmt == "cl" else x
    assert x.data_ptr() % 16 == 0
    return x


def K(id, quant, shape, fmt, calls, tags="", **call):
    """``call``: half (half_range + relu_follows), relu (relu_follows alone), bias, residual ("same", "other" strides,
    "mis" aligned 4 bytes only, "f64", "defer" / "defer_nobias" / "defer_short": a deferred shortcut whose bias is like
    the call's / absent / of other length), defer, pool, bca (bias_correct), stats (`-sm use`), tag."""
    return pytest.param(quant, shape, fmt, call, [c for c in calls.split(";") if c], tags, id=id)


CL = (2, 96, 4, 4)
ROWS = (4096, 4, 2, 2)
ROWS_OVER = (4097, 4, 2, 2)

CASES = [
    # per-channel, on-the-fly statistics: channels-last eligibility by C, pooling behind a skipped ReLU
    K("pc-c3-pool2", "pc", (2, 3, 4, 4), "cl", "fused out", "nonneg", half=True, pool=(2, 2)),
    K("pc-c3-pool3", "pc", (2, 3, 4, 4), "cl", "fused out", "nonneg", half=True, pool=(3, 3)),
    K("pc-c4-pool2", "pc", (2, 4, 4, 4), "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("pc-c4-pool3", "pc", (2, 4, 4, 4), "cl", "fused cl pool3", "nonneg pool3", half=True, pool=(3, 3)),
    K("pc-c96-pool2", "pc", CL, "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("pc-c96-pool3", "pc", CL, "cl", "fused cl pool3", "nonneg pool3", half=True, pool=(3, 3)),
    K("pc-c896-pool2", "pc", (2, 896, 4, 4), "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("pc-c896-pool3", "pc", (2, 896, 4, 4), "cl", "fused cl pool3", "nonneg pool3", half=True, pool=(3, 3)),
    K("pc-c900-pool2", "pc", (2, 900, 4, 4), "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("pc-c900-pool3", "pc", (2, 900, 4, 4), "cl", "fused cl out", "nonneg", half=True, pool=(3, 3)),
    K("pc-c2048-pool2", "pc", (2, 2048, 4, 4), "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("pc-c2048-pool3", "pc", (2, 2048, 4, 4), "cl", "fused cl out", "nonneg", half=True, pool=(3, 3)),
    K("pc-c2052-pool2", "pc", (2, 2052, 4, 4), "cl", "fused out", "nonneg", half=True, pool=(2, 2)),
    K("pc-c2052-pool3", "pc", (2, 2052, 4, 4), "cl", "fused out", "nonneg", half=True, pool=(3, 3)),
    # pooling geometry
    K("pc-oddw-pool2", "pc", (2, 96, 4, 5), "cl", "fused cl out", "nonneg", half=True, pool=(2, 2)),
    K("pc-oddw-pool3", "pc", (2, 96, 4, 5), "cl", "fused cl out", "nonneg", half=True, pool=(3, 3)),
    K("pc-oddh-pool2", "pc", (2, 96, 5, 4), "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("pc-oddh-pool3", "pc", (2, 96, 5, 4), "cl", "fused cl out", "nonneg", half=True, pool=(3, 3)),
    K("pc-h1-pool2", "pc", (2, 96, 1, 4), "cl", "fused cl out", "nonneg", half=True, pool=(2, 2)),
    K("pc-w1-pool2", "pc", (2, 96, 4, 1), "cl", "fused cl out", "nonneg", half=True, pool=(2, 2)),
    K("pc-2x2-pool3", "pc", (2, 96, 2, 2), "cl", "fused cl pool3", "nonneg pool3", half=True, pool=(3, 3)),
    K("pc-nchw-pool2", "pc", CL, "nchw", "fused out", "nonneg", half=True, pool=(2, 2)),
    K("pc-mis-pool2", "pc", CL, "mis", "fused out", "nonneg", half=True, pool=(2, 2)),
    K("pc-relu-not-skipped", "pc", CL, "cl", "fused cl out", relu=True, pool=(2, 2)),
    K("pc-pool-direct", "pc", CL, "cl", "fused cl pool2", "pool2", pool=(2, 2, "direct")),
    K("pc-pool-bias", "pc", CL, "cl", "fused bias cl pool2", "nonneg pool2", half=True, bias=True, pool=(2, 2)),
    K("pc-entropy-pool2", "pc_me", CL, "cl", "fused cl out hist", "nonneg", half=True, pool=(2, 2)),
    K("pc-pool2-residual", "pc", CL, "cl", "fused cl out res", "nonneg res", half=True, pool=(2, 2), residual="same"),
    K("pc-pool2-defer", "pc", CL, "cl", "fused cl stats", "defer nonneg", half=True, pool=(2, 2), defer=True),
    K("pcmm-pool2", "pcmm", CL, "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    K("mtd-pool2", "mtd", CL, "cl", "fused cl pool2", "nonneg pool2", half=True, pool=(2, 2)),
    # the block epilogue (residual)
    K("pc-residual", "pc", CL, "cl", "fused cl out res", "nonneg res", residual="same"),
    K("pc-residual-bias", "pc", CL, "cl", "fused bias cl out res", "nonneg res", bias=True, residual="same"),
    K("pc-residual-other-strides", "pc", CL, "cl", "fused cl out", residual="other"),
    K("pc-residual-nchw", "pc", CL, "nchw", "fused out", residual="same"),
    K("pc-residual-mis", "pc", CL, "cl", "fused cl out res", "nonneg res", residual="mis"),
    K("pc-residual-f64", "pc", CL, "cl", "fused cl out", residual="f64"),
    K("pc-residual-c2052", "pc", (2, 2052, 4, 4), "cl", "fused out", residual="same"),
    K("pc-residual-deferred", "pc", CL, "cl", "fused bias cl out rbias res rstats", "nonneg res", bias=True, residual="defer"),
    K("pc-residual-deferred-nobias", "pc", CL, "cl", "fused cl out res rstats", "nonneg res", residual="defer"),
    K("pc-residual-deferred-bias-missing", "pc", CL, "cl", "fused bias cl out", bias=True, residual="defer_nobias"),
    K("pc-residual-deferred-bias-extra", "pc", CL, "cl", "fused cl out", residual="defer_short"),
    K("pc-residual-deferred-bias-length", "pc", CL, "cl", "fused bias cl out", bias=True, residual="defer_short"),
    K("pc-entropy-residual", "pc_me", CL, "cl", "fused cl out hist", residual="same"),
    K("mtd-residual", "mtd", CL, "cl", "fused cl out res", "nonneg res", residual="same"),
    K("mtd-residual-deferred", "mtd", CL, "cl", "fused cl out", residual="defer"),
    # deferred shortcut
    K("pc-defer", "pc", CL, "cl", "fused bias cl stats", "defer", bias=True, defer=True),
    K("pc-defer-nchw", "pc", CL, "nchw", "fused bias out", bias=True, defer=True),
    K("pc-defer-mis", "pc", CL, "mis", "fused out", defer=True),
    K("pc-defer-entropy", "pc_me", CL, "cl", "fused cl out hist", defer=True),
    K("mtd-defer", "mtd", CL, "cl", "fused cl out", defer=True),
    # int8 per-sample min / max: the rows kernel (N <= 4096, per-sample elements % 4 == 0, 16-byte aligned)
    K("rows-n4096-residual", "int8", ROWS, "nchw", "fused any out res", "nonneg res", residual="same"),
    K("rows-n4097-residual", "int8", ROWS_OVER, "nchw", "fused any out", residual="same"),
    K("rows-n4096-cl-residual", "int8", ROWS, "cl", "fused any out res", "nonneg res", residual="same"),
    K("rows-n4096-defer", "int8", ROWS, "nchw", "fused any stats", "defer", defer=True),
    K("rows-n4097-defer", "int8", ROWS_OVER, "nchw", "fused any out", defer=True),
    K("rows-mis-residual", "int8", CL, "mis", "fused any out", residual="mis"),
    K("rows-mis-defer", "int8", CL, "mis", "fused any out", defer=True),
    K("rows-residual-mis", "int8", CL, "cl", "fused any out", residual="mis"),
    K("rows-residual-other-strides", "int8", CL, "cl", "fused any out", residual="other"),
    K("rows-odd-sample", "int8", (2, 3, 3, 3), "nchw", "fused any out", residual="same"),
    K("rows-odd-sample-defer", "int8", (2, 3, 3, 3), "nchw", "fused any out", defer=True),
    K("rows-entropy-residual", "int8_me", ROWS, "nchw", "fused any out", residual="same"),
    K("rows-entropy-defer", "int8_me", ROWS, "nchw", "fused any out", defer=True),
    # ... with the convolution bias: channel-fastest on channels-last memory, per-plane on NCHW memory
    K("rows-bias-cl-pool2", "int8", CL, "cl", "fused any bias bp-96 pool2", "nonneg pool2", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-cl-pool3", "int8", CL, "cl", "fused any bias bp-96 pool3", "nonneg pool3", half=True, bias=True, pool=(3, 3)),
    K("rows-bias-c4-pool3", "int8", (2, 4, 4, 4), "cl", "fused any bias bp-4 pool3", "nonneg pool3", half=True, bias=True, pool=(3, 3)),
    K("rows-bias-c896-pool3", "int8", (2, 896, 4, 4), "cl", "fused any bias bp-896 pool3", "nonneg pool3", half=True, bias=True, pool=(3, 3)),
    K("rows-bias-c900-pool2", "int8", (2, 900, 4, 4), "cl", "fused any bias bp-900 pool2", "nonneg pool2", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-c900-pool3", "int8", (2, 900, 4, 4), "cl", "fused any bias bp-900 out", "nonneg", half=True, bias=True, pool=(3, 3)),
    K("rows-bias-c2048-pool2", "int8", (2, 2048, 4, 4), "cl", "fused any bias bp-2048 pool2", "nonneg pool2", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-c2052-pool2", "int8", (2, 2052, 4, 4), "cl", "fused any out", "nonneg", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-c3-pool2", "int8", (2, 3, 4, 4), "cl", "fused any out", "nonneg", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-oddw-pool2", "int8", (2, 96, 4, 6), "cl", "fused any bias bp-96 pool2", "nonneg pool2", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-oddh-pool3", "int8", (2, 96, 5, 4), "cl", "fused any bias bp-96 out", "nonneg", half=True, bias=True, pool=(3, 3)),
    K("rows-bias-w1-pool2", "int8", (2, 96, 4, 1), "cl", "fused any bias bp-96 out", "nonneg", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-mis-pool2", "int8", CL, "mis", "fused any out", "nonneg", half=True, bias=True, pool=(2, 2)),
    K("rows-bias-nchw-pool2", "int8", CL, "nchw", "fused bias bp16 out", "nonneg", half=True, bias=True, pool=(2, 2)),
    K("rows-nobias-cl-pool2", "int8", CL, "cl", "fused any out", "nonneg", half=True, pool=(2, 2)),
    K("rows-bias-cl-residual", "int8", CL, "cl", "fused any bias bp-96 out res", "nonneg res", bias=True, residual="same"),
    K("rows-bias-cl-residual-deferred", "int8", CL, "cl", "fused any bias bp-96 out rbias res rstats", "nonneg res",
      bias=True, residual="defer"),
    K("rows-bias-cl-residual-deferred-bias-missing", "int8", CL, "cl", "fused any bias bp-96 out", bias=True,
      residual="defer_nobias"),
    K("rows-bias-cl-defer", "int8", CL, "cl", "fused any bias bp-96 stats", "defer", bias=True, defer=True),
    K("rows-bias-nchw-residual", "int8", CL, "nchw", "fused bias bp16 out", bias=True, residual="same"),
    K("rows-bias-nchw-defer", "int8", CL, "nchw", "fused bias bp16 out", bias=True, defer=True),
    K("rows-tensor-scope-bias-residual", "int8", CL, "cl", "fused any bias bp-96 out res", "nonneg res", bias=True,
      residual="same", tag=""),
    K("rows-tensor-scope-residual", "int8", CL, "cl", "fused any out", residual="same", tag=""),
    # mid-tread entropy measurement
    K("mtd-entropy-cl", "mtd_me", CL, "cl", "fused cl hist out"),
    K("mtd-entropy-nchw", "mtd_me", CL, "nchw", "fused out"),
    # `-sm use`: given parameters
    K("use-pc", "pc", CL, "cl", "quantize1 layout out", stats=True),
    K("use-pc-bias", "pc", CL, "cl", "quantize1 bias layout out", bias=True, stats=True),
    K("use-pc-residual", "pc", CL, "cl", "fused cl given out res", "nonneg res", residual="same", stats=True),
    K("use-pc-residual-other-strides", "pc", CL, "cl", "fused cl given out", residual="other", stats=True),
    K("use-pc-residual-deferred", "pc", CL, "cl", "fused bias cl given out rbias res rstats", "nonneg res", bias=True,
      residual="defer", stats=True),
    K("use-pc-residual-mis", "pc", CL, "mis", "quantize1 layout out", residual="mis", stats=True),
    K("use-pc-residual-c3", "pc", (2, 3, 4, 4), "cl", "quantize1 layout out", residual="same", stats=True),
    K("use-pc-residual-nchw", "pc", CL, "nchw", "quantize1 layout out", residual="same", stats=True),
    K("use-pc-pool2", "pc", CL, "cl", "fused cl given pool2", "nonneg pool2", half=True, pool=(2, 2), stats=True),
    K("use-pc-c896-pool3", "pc", (2, 896, 4, 4), "cl", "fused cl given pool3", "nonneg pool3", half=True, pool=(3, 3), stats=True),
    K("use-pc-c2048-pool3", "pc", (2, 2048, 4, 4), "cl", "fused cl given out", "nonneg", half=True, pool=(3, 3), stats=True),
    K("use-pc-c2052-pool2", "pc", (2, 2052, 4, 4), "cl", "quantize1 layout out", "nonneg", half=True, pool=(2, 2), stats=True),
    K("use-pc-defer", "pc", CL, "cl", "", "defer", bias=True, defer=True, stats=True),
    K("use-pc-defer-nchw", "pc", CL, "nchw", "quantize1 bias layout out", bias=True, defer=True, stats=True),
    K("use-pc-defer-mis", "pc", CL, "mis", "quantize1 layout out", defer=True, stats=True),
    K("use-pc-entropy-residual", "pc_me", CL, "cl", "quantize1 layout out", residual="same", stats=True),
    K("use-pc-entropy-defer", "pc_me", CL, "cl", "quantize1 layout out", defer=True, stats=True),
    K("use-pcmm-residual", "pcmm", CL, "cl", "fused cl given out res", "nonneg res", residual="same", stats=True),
    # `-sm use` with the activation bias correction (-bca)
    K("bca-c96", "pc", CL, "cl", "bca out relu", bca=True, stats=True),
    K("bca-c96-bias", "pc", CL, "cl", "bca bias out relu", bias=True, bca=True, stats=True),
    K("bca-c96-no-relu", "pc", CL, "cl", "bca out", bca=False, stats=True),
    K("bca-c96-nchw", "pc", CL, "nchw", "bca out relu", bca=True, stats=True),
    K("bca-c96-mis", "pc", CL, "mis", "quantize1 layout", bca=True, stats=True),
    K("bca-c3", "pc", (2, 3, 4, 4), "cl", "quantize1 layout", bca=True, stats=True),
    K("bca-c4", "pc", (2, 4, 4, 4), "cl", "bca out relu", bca=True, stats=True),
    K("bca-c900", "pc", (2, 900, 4, 4), "nchw", "bca out relu", bca=True, stats=True),
    K("bca-c2048", "pc", (2, 2048, 4, 4), "cl", "bca out relu", bca=True, stats=True),
    K("bca-c2052", "pc", (2, 2052, 4, 4), "cl", "quantize1 layout", bca=True, stats=True),
    K("bca-c2052-nchw", "pc", (2, 2052, 4, 4), "nchw", "quantize1 layout", bca=True, stats=True),
    K("bca-residual", "pc", CL, "cl", "bca out relu", bca=True, residual="same", stats=True),
    K("bca-per-tensor", "pt", CL, "cl", "bca out relu", bca=True, stats=True),
    K("use-per-tensor", "pt", CL, "cl", "quantize1 out", stats=True),
    K("use-int8", "int8", CL, "cl", "float2gemmlowp out", stats=True),
    K("use-int8-half", "int8", CL, "cl", "float2gemmlowp out", "nonneg", half=True, stats=True),
    K("use-int8-bca", "int8", CL, "cl", "float2gemmlowp", bca=True, stats=True),
]


@pytest.fixture
def rec(monkeypatch):
    r = Recorder()
    for name in ("fused", "quantize1", "quantize1_bca", "float2gemmlowp"):
        monkeypatch.setattr(ops, name, getattr(r, name))
    return r


def _residual(kind, shape, fmt, bias):
    if kind == "same":
        return _tensor(shape, fmt, seed=1)
    if kind == "other":
        return _tensor(shape, "nchw" if fmt == "cl" else "cl", seed=1)
    if kind == "mis":
        return _tensor(shape, "mis", seed=1)
    if kind == "f64":
        return _tensor(shape, fmt, seed=1).double()
    r = _tensor(shape, fmt, seed=1)
    c = shape[1]
    rbias = {"defer": None if bias is None else torch.randn(c), "defer_nobias": None, "defer_short": torch.randn(c + 4)}[kind]
    r._fq_deferred = (torch.zeros((c, L.STATS_STRIDE)), rbias)
    return r


def _tags(res, x, bias):
    tags = set()
    if getattr(res, "_fq_nonneg", None) == res._version:
        tags.add("nonneg")
    if getattr(res, "_fq_residual_fused", False):
        tags.add("res")
    if getattr(res, "_fq_pooled", False):
        tags.add("pool%d" % res._fq_pooled)
    deferred = getattr(res, "_fq_deferred", None)
    if deferred is not None:
        table, rbias = deferred
        assert res is x and table.dim() == 2 and table.shape[1] == L.STATS_STRIDE and rbias is bias
        tags.add("defer")
    return tags


@pytest.mark.parametrize("quant,shape,fmt,call,calls,tags", CASES)
def test_dispatch(rec, quant, shape, fmt, call, calls, tags):
    bits, over = QUANT[quant]
    q = IntQuantizer(bits, dict(BASE, **over))
    q.inplace = True
    q.half_range = bool(call.get("half"))
    c = shape[1]
    x = _tensor(shape, fmt)
    bias = torch.randn(c) if call.get("bias") else None
    kw = dict(bias=bias, relu_follows=bool(call.get("half") or call.get("relu")), defer=bool(call.get("defer")),
              pool=call.get("pool"), bias_correct=call.get("bca"))
    if call.get("residual"):
        kw["residual"] = _residual(call["residual"], shape, fmt, bias)
    stat_id = None
    if call.get("stats"):
        stat_id = "conv1_activation"
        q.sm = lambda: FakeStats(c if q.pcq_a else None)
    res = q(x, "conv1_activation", call.get("tag", "activation"), stat_id, None, **kw)
    assert rec.calls == [" ".join([e.split()[0]] + sorted(e.split()[1:])) for e in calls]
    assert _tags(res, x, bias) == set(tags.split())
    # the per-call inputs do not outlive the call
    assert (q._relu_follows, q._bca, q._residual, q._defer, q._pool) == (False, None, None, False, None)
