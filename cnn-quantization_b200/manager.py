"""Host-side mirror of the reference's quantization manager for the inference path
(pytorch_quantizer/quantization/inference/inference_quantization_manager.py): same tag -> quantizer table, same
call sites, same ``quantize_instant`` / ``quantize_model`` semantics, but

* call sites are PyTorch *forward hooks* on the stock ``nn.Conv2d / nn.Linear / nn.MaxPool2d / nn.AvgPool2d /
  nn.BatchNorm2d`` modules instead of the reference's class swap (``nn.Conv2d = Conv2dWithId`` ..., :518-533).
  While the manager is enabled the stock classes' ``__init__`` is wrapped only to stamp the construction-order
  id the reference's ``*WithId`` counters would have produced (:29,51,77,153,221,255);
* the quantizers are this package's ``IntQuantizer`` (one fused sm_90a launch per hooked tensor), and the
  weight bias / variance correction of ``quantize_model`` (:374-391) happens inside the weight's launch;
* nothing is a process-wide singleton: several managers can exist (one per rank / model).

``-sm no`` (on-the-fly statistics) is the mode every BASELINE config runs; ``collect`` / ``use`` (offline statistics,
SURVEY.md 8f rank 1) and ``-bca`` (rank 2, use mode only) are implemented on top of the same kernels.
"""
import argparse
import os
from itertools import count

import torch
import torch.nn as nn

from .dummy_quantizer import DummyQuantizer
from .int_quantizer import int_quantizer as _default_factory

__all__ = ["QuantizationManagerInference", "make_args", "get_params", "absorb_bn", "search_absorbe_bn",
           "resnet_mark_before_relu", "set_node_names"]

FUSED_RELU_ARCHS = ("alexnet", "vgg16", "vgg16_bn", "inception_v3")


def make_args(**over):
    """An ``args`` namespace with the reference CLI's defaults (inference/inference_sim.py:52-112) for the fields the
    manager and the quantizers read.  Extensions without a reference flag: ``stats_base_dir``, ``collect_err`` (fill the
    mse_* / cos_* columns of `-sm collect`; the name of the reference's StatisticManager argument), ``collect_mse`` (also
    write the clipping-MSE curve of every call site's quantizer in `-sm collect`, over ``mse_multipliers`` - default
    statistics.MSE_MULTIPLIERS, 0.5 .. 16 in steps of 0.125 - times the Laplace b or, with ``mse_prior="gaus"``, the std;
    `-c mse` in use mode clips at the minimum of those curves, and with ``stats_mode="no"`` each activation at the minimum
    of its own curve over the same candidates, measured in every forward), ``collect_bits`` (also write, for every call site `-sm use`
    quantizes per channel with bit allocation, the error of its quantizer on each channel at every width 0..8; needs
    ``per_channel_quant_act``, ``bit_alloc_act`` and clipping laplace, gaus or no; ``bit_alloc_prior="mse"`` (`-bap mse`) then allocates the
    widths that minimise the sum of those errors, and allocates weight widths from the weights' own errors.  With
    clipping "mse" and ``collect_mse`` - the curves clip the call sites without allocation - it measures every width at
    every ``mse_multipliers`` value instead, and `-c mse -bap mse` picks each channel's width and clipping value
    together) and
    ``measure_stats_kind`` (what `-ms` measures: "distance", the reference's default squared norms; "angle", the
    pairwise sample angles of its angle_stats module, which the reference selects by editing an import; or "noise", the
    per-sample quantization error statistics of its measure_statistics module, which the reference cannot run),
    ``clip_weight`` ("no" or "mse": quantize each output channel of a per-channel weight at the least measured squared
    error among its min/max range and the ``mse_multipliers`` clipping values under ``mse_prior``, at the widths `-baw`
    gives it or, with `-bap mse`, at the widths that minimise the sum of those least errors), ``weight_mse_report`` (a
    CSV path: one row per weight quantized under clip_weight "mse", written after quantize_model) and ``fly_bits``
    (`-baa -bap mse` with ``stats_mode="no"``: every per-channel, bit-allocated activation gets, in each forward, the
    widths that minimise the sum of its own per-channel errors - the tables collect_bits would collect under the same
    clipping rule, measured and allocated on the GPU; clipping laplace, gaus, no or mse, the last over ``mse_multipliers``
    times ``mse_prior``'s scale)."""
    d = dict(arch="resnet18", qtype=None, qweight="int8", q_off=False, clipping="no", stats_mode="no", stats_kind="mean",
             stats_folder=None, stats_batch_avg=False, kld_threshold=False, measure_stats=False,
             per_channel_quant_weights=False, per_channel_quant_act=False, bit_alloc_act=False, bit_alloc_weight=False,
             bit_alloc_rmode="round", bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None,
             bias_corr_act=False, bias_corr_weight=False, var_corr_weight=False, measure_entropy=False,
             mid_thread_quant=False, rho_act=None, rho_weight=None, preserve_zero=False, stats_base_dir=None,
             collect_err=False, measure_stats_kind="distance", collect_mse=False, mse_multipliers=None, mse_prior="laplace",
             collect_bits=False, clip_weight="no", weight_mse_report=None, fly_bits=False)
    d.update(over)
    return argparse.Namespace(**d)


def get_params(args, logger=None):
    """The ``qparams`` dict the reference builds in inference_sim.py:345-372."""
    return {
        "int": {
            "clipping": args.clipping, "stats_kind": args.stats_kind, "true_zero": args.preserve_zero,
            "kld": args.kld_threshold, "pcq_weights": args.per_channel_quant_weights,
            "pcq_act": args.per_channel_quant_act, "bit_alloc_act": args.bit_alloc_act,
            "bit_alloc_weight": args.bit_alloc_weight, "bit_alloc_rmode": args.bit_alloc_rmode,
            "bit_alloc_prior": args.bit_alloc_prior, "bit_alloc_target_act": args.bit_alloc_target_act,
            "bit_alloc_target_weight": args.bit_alloc_target_weight, "bcorr_act": args.bias_corr_act,
            "bcorr_weight": args.bias_corr_weight, "vcorr_weight": args.var_corr_weight, "logger": logger,
            "measure_entropy": args.measure_entropy, "mtd_quant": args.mid_thread_quant,
        },
        "qmanager": {"rho_act": args.rho_act, "rho_weight": args.rho_weight},
    }


# ---------------------------------------------------------------------------------------------------
# model preparation utilities (reference: utils/absorb_bn.py, utils/mark_relu.py, utils/model_naming.py)
# ---------------------------------------------------------------------------------------------------
def absorb_bn(module, bn):
    """Fold an eval-mode BatchNorm into the preceding conv / linear: w *= gamma/sigma, b = (b - mu)/sigma*gamma + beta
    (utils/absorb_bn.py:5-23; buffers stay on the module's device instead of a hard-coded .cuda())."""
    with torch.no_grad():
        w = module.weight.data
        if module.bias is None:
            module.bias = nn.Parameter(torch.zeros(w.size(0), dtype=w.dtype, device=w.device))
        b = module.bias.data
        invstd = bn.running_var.clone().add_(bn.eps).pow_(-0.5)
        shape = (w.size(0),) + (1,) * (w.dim() - 1)
        w.mul_(invstd.view(shape))
        b.add_(-bn.running_mean).mul_(invstd)
        if bn.affine:
            w.mul_(bn.weight.data.view(shape))
            b.mul_(bn.weight.data).add_(bn.bias.data)
        bn.register_buffer("running_mean", torch.zeros_like(bn.running_mean))
        bn.register_buffer("running_var", torch.ones_like(bn.running_var))
        bn.register_parameter("weight", None)
        bn.register_parameter("bias", None)
        bn.affine = False


def search_absorbe_bn(model):
    """Fold every BN that directly follows a (groups==1) conv or a linear among its siblings, mark it ``absorbed``
    (utils/absorb_bn.py:26-41)."""
    prev = None
    for m in model.children():
        is_bn = isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d))
        absorbing = (isinstance(prev, nn.Conv2d) and prev.groups == 1) or isinstance(prev, nn.Linear)
        if is_bn and absorbing:
            m.absorbed = True
            absorb_bn(prev, m)
        search_absorbe_bn(m)
        prev = m


def resnet_mark_before_relu(model):
    """Tag the convs whose output feeds a ReLU (``before_relu`` -> half_range), utils/mark_relu.py:4-29."""
    from torchvision.models.resnet import BasicBlock, Bottleneck
    root = model.module if isinstance(model, nn.DataParallel) else model
    root.conv1.before_relu = True

    def walk(m):
        for ch in m.children():
            if isinstance(ch, Bottleneck):
                for name in ("conv1", "bn1", "conv2", "bn2"):
                    getattr(ch, name).before_relu = True
            elif isinstance(ch, BasicBlock):
                ch.conv1.before_relu = True
                ch.bn1.before_relu = True
            else:
                walk(ch)

    walk(model)


def set_node_names(model):
    """``internal_name`` on every leaf module, tensorboard style (utils/model_naming.py:4-28)."""
    def type_name(m):
        return type(m).__name__.replace("WithId", "")

    def rec(parent, name):
        kids = list(parent.named_children())
        for k, m in kids:
            rec(m, name + "/" + type_name(m) + "[" + k + "]")
        if not kids:
            parent.internal_name = name

    rec(model, type_name(model))


# ---------------------------------------------------------------------------------------------------
# the manager
# ---------------------------------------------------------------------------------------------------
_STAMPED = (nn.Linear, nn.Conv2d, nn.BatchNorm2d, nn.MaxPool2d, nn.AvgPool2d)
# the call sites `-ms` measures (inference_quantization_manager.py:209-210, 247-248, 280-281): not the poolings
_MEASURED = {nn.Conv2d: "conv%d_activation", nn.Linear: "linear%d_activation", nn.BatchNorm2d: "bn%d_activation"}


def _identity_forward(x):
    return x


def _relu_forward_skipping(relu):
    """forward of an nn.ReLU that returns tensors tagged non-negative by the quantizer untouched.  The tag is the tensor's
    version counter at tagging time, so any in-place modification in between (``out += identity``) voids it."""
    orig = type(relu).forward

    def forward(x):
        if getattr(x, "_fq_nonneg", None) == x._version:
            return x
        return orig(relu, x)

    return forward


def _maxpool_forward(pool):
    """forward of an nn.MaxPool2d that pools channels-last fp32 CUDA activations with this package's kernel
    (ops.maxpool2d_cl: torch's NHWC kernel was 5 % of a ResNet-50 step and 17 % of a VGG-16 step) and leaves everything else
    to torch.  Bit-identical; the quantization hook on the module fires as before."""
    from . import ops
    orig = type(pool).forward

    def forward(x):
        pending = pool.__dict__.pop("_fq_pending", False)
        if getattr(x, "_fq_pooled", False):
            del x._fq_pooled   # consumed: the tensor object lives on (the pooling call site quantizes it in place)
            return x   # the quantization launch of the convolution in front has pooled already (IntQuantizer ``pool``)
        if pending:
            raise RuntimeError("a tensor pooled inside its quantization launch lost its tag on the way to %r" % (pool,))
        if (x.is_cuda and x.dtype == torch.float32 and not x.requires_grad and not pool.return_indices
                and not pool.ceil_mode and pool.dilation in (1, (1, 1)) and ops.nhwc(x) and x.shape[1] % 4 == 0):
            stride = pool.stride if pool.stride is not None else pool.kernel_size
            return ops.maxpool2d_cl(x, pool.kernel_size, stride, pool.padding)
        return orig(pool, x)

    return forward


def _residual_block_forward(block, bottleneck, manager):
    """forward of a torchvision BasicBlock / Bottleneck (torchvision/models/resnet.py) with the closing
    ``out += identity; out = relu(out)`` as ONE kernel (ops.add_relu_, SURVEY.md 8f rank 4: the elementwise surroundings of
    the hooked convolutions were 20 % of a step's kernel time).  Everything else goes through the block's own modules, so
    the quantization hooks fire exactly as before; results are bit-identical."""
    from . import ops

    last_conv, last_bn = (block.conv3, block.bn3) if bottleneck else (block.conv2, block.bn2)

    def forward(x):
        identity = x
        out = block.relu(block.bn1(block.conv1(x)))
        if bottleneck:
            out = block.relu(block.bn2(block.conv2(out)))
        # The shortcut depends on x only: computing it BEFORE the last convolution (torchvision does it after) lets the
        # launch that quantizes that convolution's output take it as an operand and finish the block -
        # max(quantize(conv) + identity, 0) - in its apply phase, when the folded BN behind the convolution is the
        # identity.  The set of quantize_instant calls is unchanged; the shortcut's call moves one position forward.
        early = (manager.fuse_residual_into_quant and manager.enabled and manager.bn_folding and hasattr(last_bn, "absorbed")
                 and x.is_cuda and ops.nhwc(x))
        if early:
            if block.downsample is not None:
                # ... and the shortcut convolution's output is used by that launch only: its own launch can stop after
                # the statistics phases and hand over raw tensor + parameter table (IntQuantizer ``defer``)
                ds = block.downsample
                ds_conv = ds[0] if (manager.defer_shortcut and isinstance(ds, nn.Sequential) and len(ds) == 2
                                    and isinstance(ds[0], nn.Conv2d) and hasattr(ds[1], "absorbed")) else None
                if ds_conv is not None:
                    ds_conv._fq_defer = True
                try:
                    identity = ds(x)
                finally:
                    if ds_conv is not None:
                        ds_conv.__dict__.pop("_fq_defer", None)
            last_conv._fq_residual = identity
        try:
            out = last_bn(last_conv(out))
        finally:
            last_conv.__dict__.pop("_fq_residual", None)
        if getattr(out, "_fq_residual_fused", False):
            return out
        if getattr(identity, "_fq_deferred", None) is not None:
            identity = manager.finish_deferred(identity)   # the launch above could not take it: quantize it now
        if not early and block.downsample is not None:
            identity = block.downsample(x)
        if (out.is_cuda and out.dtype == torch.float32 and identity.dtype == torch.float32 and out.shape == identity.shape
                and out.stride() == identity.stride() and ops.dense(out) and not out.requires_grad):
            return ops.add_relu_(out, identity)
        out += identity
        return block.relu(out)

    return forward


def _basic_conv_forward(block):
    """forward of a torchvision Inception ``BasicConv2d`` (conv -> bn -> ``F.relu(x, inplace=True)``) that returns tensors
    tagged non-negative by the quantizer untouched, as the hooked nn.ReLU modules do (_relu_forward_skipping): the functional
    ReLU is no module, so nothing else can skip it."""
    import torch.nn.functional as F

    def forward(x):
        x = block.bn(block.conv(x))
        if getattr(x, "_fq_nonneg", None) == x._version:
            return x
        return F.relu(x, inplace=True)

    return forward


# The branches of torchvision's Inception blocks (torchvision/models/inception.py), in the order their forward runs them:
# BasicConv2d names applied one after the other; a tuple is InceptionE's pair of convolutions on the same input whose
# outputs are concatenated; "avg" / "max" are the functional F.avg_pool2d(x, 3, 1, 1) / F.max_pool2d(x, 3, 2).
_INCEPTION_BRANCHES = {
    "InceptionA": (("branch1x1",), ("branch5x5_1", "branch5x5_2"), ("branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"),
                   ("avg", "branch_pool")),
    "InceptionB": (("branch3x3",), ("branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"), ("max",)),
    "InceptionC": (("branch1x1",), ("branch7x7_1", "branch7x7_2", "branch7x7_3"),
                   ("branch7x7dbl_1", "branch7x7dbl_2", "branch7x7dbl_3", "branch7x7dbl_4", "branch7x7dbl_5"), ("avg", "branch_pool")),
    "InceptionD": (("branch3x3_1", "branch3x3_2"), ("branch7x7x3_1", "branch7x7x3_2", "branch7x7x3_3", "branch7x7x3_4"), ("max",)),
    "InceptionE": (("branch1x1",), ("branch3x3_1", ("branch3x3_2a", "branch3x3_2b")),
                   ("branch3x3dbl_1", "branch3x3dbl_2", ("branch3x3dbl_3a", "branch3x3dbl_3b")), ("avg", "branch_pool")),
}


def _inception_block_forward(block, manager):
    """forward of a torchvision InceptionA..E whose branches write their outputs straight into the block's channels-last
    output instead of ``torch.cat``-ing them afterwards (a re-read and re-write of every branch output): the output is
    allocated once, each branch's last convolution gets its channel slice as ``_fq_out`` (the conv hook hands it to the
    quantization launch, which writes it in place), and the max-pool branch pools into its slice.  Same call sites in the
    same order, bit-identical results.  Anything but a channels-last fp32 CUDA input runs the block's own forward."""
    import torch.nn.functional as F
    from . import ops

    orig = type(block).forward
    branches = _INCEPTION_BRANCHES[type(block).__name__]

    def width(step, x):
        if step == "max":
            return x.shape[1]
        names = step if isinstance(step, tuple) else (step,)
        return sum(getattr(block, k).conv.out_channels for k in names)

    def into(name, x, sl):
        basic = getattr(block, name)
        basic.conv._fq_out = sl
        try:
            y = basic(x)
        finally:
            basic.conv.__dict__.pop("_fq_out", None)
        if y.data_ptr() != sl.data_ptr() or y.stride() != sl.stride():
            sl.copy_(y)   # the launch could not write the slice

    def forward(x):
        widths = [width(b[-1], x) for b in branches]
        if not (manager.fuse_inception_concat and manager.enabled and x.is_cuda and x.dtype == torch.float32 and ops.nhwc(x)
                and not x.requires_grad and all(ops.cl_channels_ok(c) for c in widths) and x.shape[1] % 4 == 0):
            return orig(block, x)
        n, _, h, w = x.shape
        oh, ow = ((h - 3) // 2 + 1, (w - 3) // 2 + 1) if branches[-1] == ("max",) else (h, w)
        out = torch.empty((n, sum(widths), oh, ow), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        c0 = 0
        for steps, c in zip(branches, widths):
            sl = out[:, c0:c0 + c]
            y = x
            for step in steps[:-1]:
                y = F.avg_pool2d(y, kernel_size=3, stride=1, padding=1) if step == "avg" else getattr(block, step)(y)
            last = steps[-1]
            if last == "max":
                ops.maxpool2d_cl(y, 3, 2, 0, out=sl)
            elif isinstance(last, tuple):   # InceptionE: the inner concatenation's parts go to their final places
                k0 = 0
                for name in last:
                    k = getattr(block, name).conv.out_channels
                    into(name, y, sl[:, k0:k0 + k])
                    k0 += k
            else:
                into(last, y, sl)
            c0 += c
        return out

    return forward


class QuantizationManagerInference(object):
    """``with QuantizationManagerInference(args, qparams) as qm: model = build(); qm.attach(model); qm.quantize_model(model)``.

    ``quantizer_factory(qtype, quant_params)`` defaults to this package's CUDA ``int_quantizer``; tests and the CPU
    baseline inject the oracle's factory to run the very same call sites on CPU."""

    def __init__(self, args, qparams, quantizer_factory=None):
        self.args = args
        self.verbose = False
        self.quantize = args.qtype is not None
        self.disable_quantization = args.q_off
        self.enabled = False
        self.bn_folding = False
        self.bcorr_act = args.bias_corr_act
        self.bcorr_weight = args.bias_corr_weight
        self.vcorr_weight = args.var_corr_weight
        if args.stats_mode not in ("no", "collect", "use"):
            raise ValueError("stats_mode must be one of no / collect / use, got %r" % (args.stats_mode,))
        self.stats_mode = args.stats_mode
        self._factory = quantizer_factory or _default_factory
        # extensions of this package's CUDA quantizer (a foreign factory - the CPU oracle - gets plain reference calls)
        self._native = quantizer_factory is None
        if not self._native and self.stats_mode != "no":
            raise NotImplementedError("offline statistics run through this package's CUDA quantizers only")
        self._fuse_weight_correction = self._native
        # run hooked convolutions bias-free and add the bias inside the fused kernel (statistics collection wants the
        # tensor the network actually produces, so not in collect mode)
        self.fuse_conv_bias = self._native and self.stats_mode != "collect"
        # a half-range / force-positive quantization returns values >= 0 (offset 0 -> zero point 0): the ReLU that
        # follows it is the identity, so the hooked ReLU modules skip the pass over tensors tagged by the conv hook
        self.skip_redundant_relu = self._native
        # the `out += identity; relu` that closes a torchvision ResNet block runs as one fused kernel
        self.fuse_residual_relu = self._native
        # ... and, where the quantization launch of the block's last convolution can take the shortcut as an operand, inside
        # that launch (channels-last per-channel activations with on-the-fly statistics)
        self.fuse_residual_into_quant = self._native
        # ... and the shortcut convolution of a down-sampling block runs statistics-only, quantized on the fly there
        self.defer_shortcut = self._native
        # a 2x2 / stride-2 max pooling behind a hooked convolution (+ skipped ReLU) runs inside that convolution's launch
        self.fuse_pool_into_quant = self._native
        # channels-last max pooling in front of the `activation_pooling` call site runs on this package's kernel
        self.fast_maxpool = self._native
        # the branches of a torchvision Inception block write their (quantized) outputs into the block's output directly,
        # without the closing torch.cat (not with `-bca`, whose launch writes no channel slice)
        self.fuse_inception_concat = self._native and not self.bcorr_act
        self.inplace_activations = self._native
        # `-ms` (inference_quantization_manager.py:320-323): the per-sample squared norm of the tensor every conv / linear /
        # non-absorbed BN call site hands on.  Three launches never write that tensor - the block epilogue writes
        # max(q + identity, 0), a deferred shortcut is quantized only inside the consuming launch, a pooling launch writes
        # the pooled quarter - so they are switched off; each is bit-identical to its unfused form.
        # The noise kind also measures the tensor the quantizer was handed, so activations are quantized out of place and
        # that tensor survives the launch; the convolution bias stays fused and is passed to the measurement.
        # `clip_weight="mse"`: measured clipping of the per-channel weights, shared by the weight quantizers
        from .int_quantizer import WeightMse, refuse_clip_weight
        clip_weight = getattr(args, "clip_weight", "no")
        refuse_clip_weight(clip_weight, args.per_channel_quant_weights, args.mid_thread_quant, qweight=args.qweight,
                           native=self._native)
        report = getattr(args, "weight_mse_report", None)
        if report is not None and clip_weight != "mse":
            raise ValueError("weight_mse_report reports the weights quantized under clip_weight='mse'")
        # the clipping candidates (mse_multipliers / mse_prior) every measurement of this run shares: checked where the
        # first one needs them (``_mse_candidates``)
        self._mse_set = None
        self.weight_mse = None
        if clip_weight == "mse":
            self.weight_mse = WeightMse(self._mse_candidates(), report=report)
        # `-c mse` with on-the-fly statistics: every activation is clipped at the minimum of its own clipping-MSE curve
        # over these candidates, measured and chosen on the device in each forward
        self.fly_mse = None
        if args.clipping == "mse" and self.stats_mode == "no":
            self.fly_mse = self._mse_candidates()
            if args.measure_entropy and not getattr(args, "mid_thread_quant", False):
                raise NotImplementedError("-c mse with -sm no does not measure entropy (-me): use -sm use with curves "
                                          "collected with collect_mse=True")
        self.measure_stats = None
        kind = getattr(args, "measure_stats_kind", "distance")
        if kind not in ("distance", "angle", "noise"):
            raise ValueError("measure_stats_kind must be 'distance', 'angle' or 'noise', got %r" % (kind,))
        if args.measure_stats:
            if kind == "noise" and self.stats_mode == "collect":
                raise ValueError("measure_stats_kind='noise' measures quantization noise: collect mode quantizes nothing")
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                raise NotImplementedError("-ms with several ranks: per-rank shards would put the rows out of sample order")
            from .statistics import AngleStatistics, MeasureStatistics, NoiseStatistics
            cls = {"distance": MeasureStatistics, "angle": AngleStatistics, "noise": NoiseStatistics}[kind]
            self.measure_stats = cls(args.arch, getattr(args, "stats_base_dir", None))
            self.fuse_residual_into_quant = self.defer_shortcut = self.fuse_pool_into_quant = False
            self.fuse_inception_concat = False   # the hooked output is the tensor -ms measures; keep torch.cat's
            if kind == "noise":
                self.inplace_activations = False
        # `collect_err`: the collect hooks hand each tensor's use-mode quantizer settings to save_tensor_stats, which fills
        # the mse_* / cos_* columns `-c mix` chooses by
        self.collect_err = bool(getattr(args, "collect_err", False))
        if self.collect_err and (self.stats_mode != "collect" or args.qtype is None):
            raise ValueError("collect_err fills error columns of -sm collect for the bit widths of -qtype: it needs "
                             "stats_mode='collect' and a qtype (got stats_mode=%r, qtype=%r)" % (self.stats_mode, args.qtype))
        # `collect_mse`: the collect hooks also measure each tensor's clipping-MSE curve with the same quantizer settings
        self.collect_mse = bool(getattr(args, "collect_mse", False))
        if self.collect_mse and (self.stats_mode != "collect" or args.qtype is None):
            raise ValueError("collect_mse measures the clipping-MSE curves of -sm collect for the bit widths of -qtype: it "
                             "needs stats_mode='collect' and a qtype (got stats_mode=%r, qtype=%r)" % (self.stats_mode, args.qtype))
        self.clip_mse = None
        # `collect_bits`: the collect hooks also measure the per-channel error tables `-bap mse` allocates from
        self.collect_bits = bool(getattr(args, "collect_bits", False))
        from .statistics import BIT_RULES, refuse_bap_mse
        if self.collect_bits:
            missing = [what for what, ok in (("stats_mode='collect'", self.stats_mode == "collect"),
                                              ("a qtype", args.qtype is not None),
                                              ("per_channel_quant_act", args.per_channel_quant_act),
                                              ("bit_alloc_act", args.bit_alloc_act),
                                              ("clipping laplace, gaus or no (or mse with collect_mse)",
                                               args.clipping in BIT_RULES and (args.clipping != "mse" or self.collect_mse)))
                       if not ok]
            if missing:
                raise ValueError("collect_bits measures the per-channel error tables of -sm collect: it needs %s"
                                 % ", ".join(missing))
        bap_mse = getattr(args, "bit_alloc_prior", None) == "mse"
        # `fly_bits`: `-baa -bap mse` with on-the-fly statistics - each activation's tables measured and allocated on the
        # device in every forward
        self.fly_bits = bool(getattr(args, "fly_bits", False))
        if bap_mse:   # a k*std rule is refused by the quantizer, at the call sites that would allocate under it
            refuse_bap_mse(kld=args.kld_threshold, clipping="mix" if args.clipping == "mix" else None,
                           mid_tread=getattr(args, "mid_thread_quant", False),
                           needs_use=args.bit_alloc_act and self.stats_mode == "no" and not self.fly_bits,
                           collect=args.bit_alloc_act and (self.collect_err or self.collect_mse))
        if self.fly_bits:
            missing = [what for what, ok in (("stats_mode='no'", self.stats_mode == "no"),
                                              ("a qtype", args.qtype is not None),
                                              ("per_channel_quant_act", args.per_channel_quant_act),
                                              ("bit_alloc_act", args.bit_alloc_act),
                                              ("bit_alloc_prior='mse'", bap_mse),
                                              ("clipping laplace, gaus, no or mse", args.clipping in BIT_RULES),
                                              ("this package's quantizers (no quantizer_factory)", self._native))
                       if not ok]
            if missing:
                raise ValueError("fly_bits allocates each activation's widths from its own per-channel error tables in "
                                 "every forward: it needs %s" % ", ".join(missing))
            if args.measure_entropy:
                raise NotImplementedError("-baa -bap mse on the fly (fly_bits) does not measure entropy (-me)")
        self.bit_mse = None
        # offline statistics (inference_quantization_manager.py:299-318)
        self.stats_manager = None
        self._sm_tensor = self._sm_channel = None
        if self.stats_mode != "no":
            from .statistics import StatisticManager, StatisticManagerPerChannel
            sf = args.stats_folder if args.stats_folder is not None else args.arch
            if args.kld_threshold:
                sf += "_kld_" + args.qtype   # inference_quantization_manager.py:300-301
            base = getattr(args, "stats_base_dir", None)
            if self.stats_mode == "collect":
                print("Collecting statistics...")
                if args.per_channel_quant_act:
                    self.stats_manager = StatisticManagerPerChannel(sf, load_stats=False, batch_avg=args.stats_batch_avg,
                                                                    collect_err=self.collect_err, base_dir=base)
                else:
                    self.stats_manager = StatisticManager(sf, load_stats=False, kld_threshold=args.kld_threshold,
                                                          batch_avg=args.stats_batch_avg, base_dir=base)
                if self.collect_mse:
                    from .statistics import ClipMseStatistics
                    self.clip_mse = ClipMseStatistics(sf, self._mse_candidates(), base_dir=base)
                if self.collect_bits:
                    from .statistics import BitMseStatistics
                    self.bit_mse = BitMseStatistics(sf, args.clipping, base_dir=base,
                                                    multipliers=self._mse_candidates() if args.clipping == "mse" else None)
            else:
                if bap_mse:   # read on first use: a missing layer raises KeyError naming collect_bits there
                    from .statistics import BitMseStatistics
                    self.bit_mse = BitMseStatistics(sf, base_dir=base, load=True)
                    if args.clipping == "mse" and args.bit_alloc_act and not os.path.exists(self.bit_mse.path):
                        # without joint tables the only combination left is -c mse's curves at separately measured
                        # widths, which is not implemented: -c mse -bap mse picks width and clipping value together
                        raise NotImplementedError("-c mse -baa -bap mse picks each channel's width and clipping value "
                                                  "from joint tables, and there are none at %s: collect them under -c mse "
                                                  "with collect_bits=True and collect_mse=True" % self.bit_mse.path)
                if args.per_channel_quant_act:
                    self._sm_channel = StatisticManagerPerChannel(sf, load_stats=True, base_dir=base)
                self._sm_tensor = StatisticManager(sf, load_stats=True, base_dir=base)
                if args.clipping == "mse":   # read on first use: a missing file raises KeyError naming collect_mse there
                    from .statistics import ClipMseStatistics
                    self.clip_mse = ClipMseStatistics(sf, base_dir=base, load=True)
        self.fused_relu = args.arch is not None and (args.arch in FUSED_RELU_ARCHS or "squeezenet" in args.arch)
        self.ignore_ids = []
        self.quantizers = {}
        self.quantizer_default = None
        self.calls = []          # (id, tag, half_range, shape) of every quantize_instant while `record` is set
        self.record = False
        self._hooks = []
        self._patched = []
        self._pool_marked = []
        self._debiased = []
        self._orig_init = {}
        self._counters = {}
        if self.quantize:
            self.__fill_quantizers__(args.qtype, qparams, args.arch, args.qweight)
            self.quantizer_default = self._load("int8", qparams)
            if self.weight_mse is not None:
                for tag in ("weight", "weight_classifier"):
                    self.quantizers[tag].clip_weight, self.quantizers[tag].weight_mse = "mse", self.weight_mse
            if self.fly_mse is not None:
                for q in list(self.quantizers.values()) + [self.quantizer_default]:
                    if getattr(q, "clipping", None) == "mse":
                        q.mse_candidates = self.fly_mse
            if self.fly_bits:   # the quantizers take the route at the per-channel, bit-allocated activation call sites
                for q in list(self.quantizers.values()) + [self.quantizer_default]:
                    if hasattr(q, "fly_bits"):
                        q.fly_bits = True
            if self.stats_mode == "use":
                # which statistics each tag reads (IntQuantizer.__init__ :88 + the overrides of __fill_quantizers__)
                per_tensor = lambda: self._sm_tensor
                per_channel = (lambda: self._sm_channel) if self._sm_channel is not None else per_tensor
                for tag, q in list(self.quantizers.items()) + [("", self.quantizer_default)]:
                    if isinstance(q, DummyQuantizer):
                        continue
                    q.sm = per_channel if tag in ("activation", "weight", "weight_classifier", "") else per_tensor
                    q.mse_curves = self.clip_mse
                    q.bit_tables = self.bit_mse
            if self.inplace_activations:
                for tag, q in list(self.quantizers.items()) + [("", self.quantizer_default)]:
                    if tag.startswith("activation") or tag in ("", "ignored"):
                        q.inplace = True
            if args.qtype == "int4":
                self.set_8bit_list(["conv%d_activation" % i for i in [0]])  # createTruncationManager, :334-340

    # -- quantizer table (TruncationOpManagerInference.__fill_quantizers__, :407-476) ----------------
    def _mse_candidates(self):
        """The run's statistics.MseCandidates of mse_multipliers / mse_prior, made and checked on first use."""
        if self._mse_set is None:
            from .statistics import MseCandidates
            self._mse_set = MseCandidates.of(getattr(self.args, "mse_multipliers", None),
                                             getattr(self.args, "mse_prior", "laplace"))
        return self._mse_set

    def _load(self, qtype, qparams):
        name = qtype.rstrip("1234567890")
        if name != "int":
            raise NotImplementedError("qtype %r: only the int quantizer is on the hot path" % qtype)
        return self._factory(qtype, qparams[name] if name in qparams else {})

    def __fill_quantizers__(self, qtype, qparams, arch=None, qweight="int8"):
        q = self._load("int8", qparams)
        q.clipping, q.kld, q.pcq_w, q.pcq_a, q.stats_kind, q.measure_entropy = "no", False, False, False, "max", False
        self.quantizers["activation_classifier"] = q

        if qweight == "f32":
            q = DummyQuantizer()
        else:
            q = self._load(qweight, qparams)
            q.pcq_a, q.clipping, q.kld, q.stats_kind = False, "no", False, "max"
        self.quantizers["weight"] = q

        q = self._load("int8", qparams)
        q.pcq_a, q.clipping, q.kld, q.stats_kind, q.measure_entropy = False, "no", False, "max", False
        self.quantizers["weight_classifier"] = q

        self.quantizers["bias"] = DummyQuantizer()

        q = self._load("int8", qparams)
        q.pcq_w, q.pcq_a, q.clipping, q.kld = False, False, "no", False
        self.quantizers["ignored"] = q

        q = self._load(qtype, qparams)
        q.force_positive, q.pcq_w = self.fused_relu, False
        self.quantizers["activation"] = q

        q = self._load(qtype, qparams)
        q.force_positive, q.pcq_w, q.pcq_a = self.fused_relu, False, False
        self.quantizers["activation_linear"] = q

        q = self._load("int8", qparams)
        q.pcq_w, q.pcq_a, q.clipping, q.kld, q.measure_entropy = False, False, "no", False, False
        self.quantizers["activation_pooling"] = q

    def get_quantizer(self, tag, tensor=None):
        return self.quantizers[tag] if tag in self.quantizers else self.quantizer_default

    def set_8bit_list(self, ignore_ids):
        self.ignore_ids = ignore_ids

    def reset_counters(self):
        pass

    # -- enable / disable: stamp construction order like the reference's class-level counters --------------
    def enable(self):
        if not self.quantize:
            return
        self.enabled = not self.disable_quantization
        if self._orig_init:
            return
        self._counters = {cls: count(0) for cls in _STAMPED}
        for cls in _STAMPED:
            orig = cls.__init__
            self._orig_init[cls] = orig

            def stamped(mod, *a, __orig=orig, __cls=cls, **k):
                __orig(mod, *a, **k)
                if type(mod) is __cls or not hasattr(mod, "_fq_id"):
                    mod._fq_id = next(self._counters[__cls])

            cls.__init__ = stamped

    def stop_stamping(self):
        """Restore the stock constructors (ids already stamped stay); quantization stays enabled."""
        for cls, orig in self._orig_init.items():
            cls.__init__ = orig
        self._orig_init = {}

    def disable(self):
        self.enabled = False
        self.stop_stamping()

    def __enter__(self):
        self.enable()
        return self

    def __exit__(self, *exc):
        self.disable()
        self.detach()
        if self.stats_manager is not None:
            self.stats_manager.__exit__()  # collect mode: write the CSV / pickle files
        if self.clip_mse is not None:
            self.clip_mse.__exit__()       # collect_mse: clip_mse.pkl and curve.csv
        if self.bit_mse is not None:
            self.bit_mse.__exit__()        # collect_bits: bit_mse.pkl and alloc.csv
        if self.measure_stats is not None:
            self.measure_stats.__exit__()  # -ms: write distance.csv (angle.pkl, noise/<id>.csv with the other kinds)

    # -- call sites: forward hooks reproducing the *WithId.forward bodies (:58-74, :84-101, :162-217, :227-250, :262-283)
    def attach(self, model):
        """Register the forward hooks.  Modules built outside ``enable()`` get ids in ``model.modules()`` order."""
        fallback = {cls: count(0) for cls in _STAMPED}
        if self.fuse_residual_relu and self.enabled and self.stats_mode != "collect":
            try:
                from torchvision.models.resnet import BasicBlock, Bottleneck
            except ImportError:  # pragma: no cover
                BasicBlock = Bottleneck = ()
            for m in model.modules():
                if type(m) in (BasicBlock, Bottleneck) and type(getattr(m, "relu", None)) is nn.ReLU:
                    m.forward = _residual_block_forward(m, type(m) is Bottleneck, self)
                    self._patched.append(m)
        if self.enabled and self.stats_mode != "collect" and self.measure_stats is None:
            try:
                from torchvision.models import inception as tv_inception
            except ImportError:  # pragma: no cover
                tv_inception = None
            for m in model.modules() if tv_inception is not None else ():
                if type(m) is tv_inception.BasicConv2d and self.skip_redundant_relu:
                    m.forward = _basic_conv_forward(m)
                    self._patched.append(m)
                elif self.fuse_inception_concat and type(m).__name__ in _INCEPTION_BRANCHES and type(m) is getattr(tv_inception, type(m).__name__):
                    m.forward = _inception_block_forward(m, self)
                    self._patched.append(m)
        if self.fuse_pool_into_quant and self.fast_maxpool and self.skip_redundant_relu and self.enabled and self.stats_mode in ("no", "use"):
            two = lambda v: (v, v) if isinstance(v, int) else tuple(v)

            def pool_kind(pm):
                """2: 2x2 / stride 2; 3: 3x3 / stride 2 / padding 1; None: not a pooling the quantization launch can do"""
                if type(pm) is not nn.MaxPool2d or two(pm.dilation) != (1, 1) or pm.ceil_mode or pm.return_indices:
                    return None
                geo = (two(pm.kernel_size), two(pm.stride if pm.stride is not None else pm.kernel_size), two(pm.padding))
                return {((2, 2), (2, 2), (0, 0)): 2, ((3, 3), (2, 2), (1, 1)): 3}.get(geo)

            def mark(conv, pm, direct):
                if type(conv) is nn.Conv2d and pool_kind(pm) is not None:
                    conv._fq_pool_module = (pm, direct, pool_kind(pm))
                    self._pool_marked.append(conv)

            for seq in model.modules():
                if isinstance(seq, nn.Sequential):   # VGG: Conv2d, [BatchNorm2d (folded away),] [ReLU,] MaxPool2d
                    kids = [k for k in seq.children()
                            if not (self.bn_folding and type(k) is nn.BatchNorm2d and hasattr(k, "absorbed"))]
                    for i, conv in enumerate(kids):
                        nxt = kids[i + 1:i + 3]
                        if len(nxt) >= 1 and type(nxt[0]) is nn.MaxPool2d:
                            mark(conv, nxt[0], True)
                        elif len(nxt) == 2 and type(nxt[0]) is nn.ReLU and type(nxt[1]) is nn.MaxPool2d:
                            mark(conv, nxt[1], False)
                elif type(seq).__name__ == "ResNet" and all(hasattr(seq, a) for a in ("conv1", "bn1", "relu", "maxpool")):
                    # torchvision ResNet._forward_impl: conv1 -> bn1 -> relu -> maxpool; bn1 must be folded away
                    if self.bn_folding and hasattr(seq.bn1, "absorbed") and type(seq.relu) is nn.ReLU:
                        mark(seq.conv1, seq.maxpool, False)
        for m in model.modules():
            if self.fast_maxpool and self.enabled and type(m) is nn.MaxPool2d:
                m.forward = _maxpool_forward(m)
                self._patched.append(m)
            if self.skip_redundant_relu and self.enabled and type(m) is nn.ReLU and self.stats_mode != "collect":
                m.forward = _relu_forward_skipping(m)
                self._patched.append(m)
                continue
            cls = next((c for c in _STAMPED if type(m) is c), None)
            if cls is None:
                continue
            if not hasattr(m, "_fq_id"):
                m._fq_id = next(fallback[cls])
            if cls is nn.BatchNorm2d and self.bn_folding and hasattr(m, "absorbed"):
                # :264-265: an absorbed BN returns its input untouched; do not even run the (identity) normalisation
                m.forward = _identity_forward
                self._patched.append(m)
                continue
            if cls is nn.Conv2d and self.fuse_conv_bias and self.enabled and m.bias is not None:
                # the convolution runs bias-free; the (folded-BN) bias is added inside the fused quantization kernel.  The
                # vector stays with the module as a (non-persistent) BUFFER, so .to() / .cuda() / DataParallel replicas
                # carry it along; detach() puts the parameter back, on whatever device the module lives by then.
                m._fq_bias_param = m.bias
                m.bias = None
                m.register_buffer("_fq_bias", m._fq_bias_param.data, persistent=False)
                self._debiased.append(m)
            hook = {nn.Conv2d: self._conv_hook, nn.Linear: self._linear_hook, nn.MaxPool2d: self._maxpool_hook,
                    nn.AvgPool2d: self._avgpool_hook, nn.BatchNorm2d: self._bn_hook}[cls]
            if self.measure_stats is not None and cls in _MEASURED:
                hook = self._measuring(hook, _MEASURED[cls])
            self._hooks.append(m.register_forward_hook(hook))
        return model

    def detach(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []
        for m in self._patched:
            m.__dict__.pop("forward", None)
        self._patched = []
        for m in self._pool_marked:
            m.__dict__.pop("_fq_pool_module", None)
        self._pool_marked = []
        for m in self._debiased:
            param = m._fq_bias_param
            param.data = m._fq_bias.data   # follows the module if it moved / changed dtype while attached
            del m._buffers["_fq_bias"]
            m._non_persistent_buffers_set.discard("_fq_bias")
            del m._fq_bias_param
            m.bias = param
        self._debiased = []

    def _measuring(self, hook, id_format):
        """``hook`` followed by the `-ms` measurement of what the call site hands on: the hook's result, or ``out`` where
        the hook leaves it (collect mode, quantization disabled).  Measured whether or not quantization is enabled, as the
        reference's *WithId modules do; an absorbed BN (the identity) is not a measured site.  The noise kind measures
        that tensor against ``out`` (plus the convolution bias the launch added to it), with ``inputs[0]`` and the
        module's weight (a BN's gamma)."""
        from . import ops
        from .statistics import NoiseStatistics
        noise = isinstance(self.measure_stats, NoiseStatistics)

        def measured(m, inputs, out):
            res = hook(m, inputs, out)
            if not (isinstance(m, nn.BatchNorm2d) and self.bn_folding and hasattr(m, "absorbed")):
                handed_on, id = out if res is None else res, id_format % m._fq_id
                if noise:
                    bias = getattr(m, "_fq_bias", None)   # a fused convolution bias: out is bias-free
                    period = 0 if bias is None else (-out.shape[1] if ops.nhwc(out) else out[0, 0].numel())
                    self.measure_stats.save_measure(out, handed_on, inputs[0], m.weight, id, bias=bias, bias_period=period)
                else:
                    self.measure_stats.save_measure(handed_on, id)
            return res

        return measured

    def _clip_err(self, out, tag, stat_id, half_range, name):
        """``save_tensor_stats`` kwargs of a collect call site: with collect_err, the settings (``clip_err_config``, at
        most 8 bits) of the quantizer quantize_instant picks for the same call in `-sm use` (``tag``, the 8-bit
        ``ignored`` list, ``half_range``) on this tensor ``out``.  With collect_mse, the call site's clipping-MSE curve
        is measured here, with the same settings (``name``: the internal name save_tensor_stats records).  With
        collect_bits, a call site it would quantize per channel with bit allocation also gets its per-channel error
        tables measured."""
        if not (self.collect_err or self.collect_mse or self.collect_bits):
            return {}
        q = self.get_quantizer("ignored" if stat_id in self.ignore_ids else tag)
        cfg = q.clip_err_config(out, half_range)._replace(num_bits=min(q.num_bits, 8))
        if self.collect_mse:
            self.clip_mse.save_curve(out, name, stat_id, cfg)
        if self.collect_bits:
            self.bit_mse.save_table(out, name, stat_id, cfg)
        return {"clip_err": cfg} if self.collect_err else {}

    def _stat_id(self, activation_id):
        return activation_id if self.stats_mode == "use" else None

    def _conv_hook(self, m, inputs, out):
        bias = getattr(m, "_fq_bias", None)
        if not self.enabled:
            return None if bias is None else out + bias.view(1, -1, 1, 1)
        activation_id = "conv%d_activation" % m._fq_id
        tag = "activation_classifier" if out.shape[1] == 1000 else "activation"
        half_range = hasattr(m, "before_relu")
        if self.stats_mode == "collect":
            name = getattr(m, "internal_name", activation_id)
            self.stats_manager.save_tensor_stats(out, name, activation_id,
                                                 **self._clip_err(out, tag, activation_id, half_range, name))
            return None
        extra = {} if bias is None else {"bias": bias}
        if self.stats_mode == "use" and self.bcorr_act:
            # `-bca` (:180-196): the correction runs inside the quantizer's given-parameter launch
            return self.quantize_instant(out, activation_id, tag, stat_id=activation_id, half_range=half_range,
                                         verbose=self.verbose, bias_correct=bool(half_range or self.fused_relu), **extra)
        if self.skip_redundant_relu and (half_range or self.fused_relu) and tag == "activation" and not self.bcorr_act:
            extra["relu_follows"] = True   # the quantizer tags the result _fq_nonneg; the hooked ReLU then returns it untouched
        residual = m.__dict__.get("_fq_residual")
        if residual is not None and self._native and tag == "activation":
            extra["residual"] = residual
        pm = m.__dict__.get("_fq_pool_module")
        if pm is not None and self._native and tag == "activation" and (pm[1] or extra.get("relu_follows")):
            res = self.quantize_instant(out, activation_id, tag, stat_id=self._stat_id(activation_id), half_range=half_range, verbose=self.verbose,
                                        pool=(pm[2], pm[2], "direct") if pm[1] else (pm[2], pm[2]), **extra)
            # the pooling module must find the tag when the launch has pooled (it raises otherwise); a stale flag of an
            # aborted forward is overwritten here
            pm[0]._fq_pending = bool(getattr(res, "_fq_pooled", False))
            return res
        into = m.__dict__.get("_fq_out")
        if into is not None and self._native and tag == "activation":
            extra["out"] = into   # an Inception branch: its part of the block's output, written in place where the launch can
        if m.__dict__.get("_fq_defer") and self._native and tag == "activation":
            res = self.quantize_instant(out, activation_id, tag, stat_id=self._stat_id(activation_id), half_range=half_range,
                                        verbose=self.verbose, defer=True, **extra)
            if getattr(res, "_fq_deferred", None) is not None:
                res._fq_redo = (activation_id, tag, half_range, extra)
            return res
        return self.quantize_instant(out, activation_id, tag, stat_id=self._stat_id(activation_id), half_range=half_range,
                                     verbose=self.verbose, **extra)

    def finish_deferred(self, tensor):
        """Quantize a tensor whose launch was deferred (IntQuantizer ``defer``) after all: the call that should have taken
        it as its residual did not fuse.  Same quantizer, same arguments; not recorded as a second call."""
        activation_id, tag, half_range, extra = tensor._fq_redo
        del tensor._fq_deferred, tensor._fq_redo
        stat_id = self._stat_id(activation_id)
        ignore = stat_id is not None and any(l == stat_id for l in self.ignore_ids)
        q = self.get_quantizer("ignored" if ignore else tag)
        q.half_range = half_range
        return q(tensor, activation_id, tag, stat_id, None, **extra)

    def _linear_hook(self, m, inputs, out):
        if not self.enabled:
            return None
        classifier = m.weight.shape[0] == 1000
        activation_id = "linear%d_activation" % m._fq_id
        tag = "activation_classifier" if classifier else "activation_linear"
        half_range = hasattr(m, "before_relu") if not classifier else False
        if self.stats_mode == "collect":
            self.stats_manager.save_tensor_stats(out, tag, activation_id, force_global_min_max=("classifier" in tag),
                                                 **self._clip_err(out, tag, activation_id, half_range, tag))
            return None
        return self.quantize_instant(out, activation_id, tag, stat_id=self._stat_id(activation_id), half_range=half_range,
                                     verbose=self.verbose)

    def _maxpool_hook(self, m, inputs, out):
        if not self.enabled:
            return None
        out_id = "maxpool%d_out" % m._fq_id
        if self.stats_mode == "collect":
            self.stats_manager.save_tensor_stats(out, "activation_pooling", out_id,
                                                 **self._clip_err(out, "activation_pooling", out_id, False,
                                                                  "activation_pooling"))
            return None
        return self.quantize_instant(out, out_id, "activation_pooling", stat_id=self._stat_id(out_id), verbose=self.verbose)

    def _avgpool_hook(self, m, inputs, out):
        if not self.enabled:
            return None
        out_id = "avgpool%d_out" % m._fq_id
        tag_act = "activation_classifier" if out.shape[1] == 1000 else "activation_pooling"
        if self.stats_mode == "collect":
            self.stats_manager.save_tensor_stats(out, tag_act, out_id, **self._clip_err(out, "", out_id, False, tag_act))
            return None
        # the reference passes the tag in the id slot here (:96,:99): the tensor goes through the DEFAULT quantizer
        return self.quantize_instant(out, tag_act, stat_id=self._stat_id(out_id), verbose=self.verbose)

    def _bn_hook(self, m, inputs, out):
        if self.bn_folding and hasattr(m, "absorbed"):
            return inputs[0]  # :264-265: an absorbed BN is the identity
        if not self.enabled:
            return None
        activation_id = "bn%d_activation" % m._fq_id
        if self.stats_mode == "collect":
            self.stats_manager.save_tensor_stats(out, "activation", activation_id,
                                                 **self._clip_err(out, "", activation_id, hasattr(m, "before_relu"),
                                                                  "activation"))
            return None
        # same argument-order slip as the reference (:275,:278): id="activation", tag="" -> default quantizer
        return self.quantize_instant(out, "activation", stat_id=self._stat_id(activation_id),
                                     half_range=hasattr(m, "before_relu"), verbose=self.verbose)

    # -- quantize_instant (:549-562) ------------------------------------------------------------------------
    def quantize_instant(self, tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False,
                         **extra):
        ignore = stat_id is not None and any(l == stat_id for l in self.ignore_ids)
        qtag = "ignored" if ignore else tag
        q = self.get_quantizer(qtag)
        q.half_range = half_range
        if verbose:
            print("Quantize {0:21} | Id - {1:18} | {2:} | {3:}".format(tag, str(stat_id), str(q), str(tensor.device)))
        if self.record:
            self.calls.append((id, tag, bool(half_range), tuple(tensor.shape)))
        if isinstance(q, DummyQuantizer):
            return q(tensor, id, tag, stat_id, override_att)
        return q(tensor, id, tag, stat_id, override_att, **extra)

    # -- quantize_model (:352-393) ---------------------------------------------------------------------------
    def quantize_model(self, model):
        if self.stats_mode == "collect":
            return  # :353-354: weights stay fp32 while statistics are collected
        import torchvision
        inception = isinstance(model, torchvision.models.Inception3)
        corr = (bool(self.bcorr_weight), bool(self.vcorr_weight))
        for n, m in model.named_modules():
            weight_q = None
            extra = {"weight_correction": corr} if (self._fuse_weight_correction and any(corr)) else {}
            if isinstance(m, nn.Conv2d):
                first8 = (inception and n in ("Conv2d_1a_3x3.conv", "Conv2d_2a_3x3.conv")) or m.weight.shape[1] == 3
                weight_q = self.quantize_instant(m.weight.data, n + ".weight", "weight",
                                                 override_att=("num_bits", 8) if first8 else None, verbose=self.verbose,
                                                 **extra)
            elif isinstance(m, nn.Linear):
                tag = "weight_classifier" if m.weight.shape[0] == 1000 else "weight"
                weight_q = self.quantize_instant(m.weight.data, n + ".weight", tag, verbose=self.verbose, **extra)
            if weight_q is None:
                continue
            if any(corr) and not extra:
                weight_q = self._weight_correction_torch(m.weight.data, weight_q, *corr)
            m.weight.data = weight_q
        if self.weight_mse is not None:
            self.weight_mse.finish()   # the one read-back of clip_weight="mse": its report and its non-finite flag

    @staticmethod
    def _weight_correction_torch(w, w_q, bias_corr, var_corr):
        """:374-391 as stock torch ops: only used when a foreign quantizer factory (the CPU oracle) is injected."""
        bshape = (-1, 1, 1, 1) if w_q.dim() == 4 else (-1, 1)
        m_q = w_q.view(w_q.shape[0], -1).mean(-1).view(bshape)
        m_o = w.view(w.shape[0], -1).mean(-1).view(bshape)
        if var_corr:
            eps = torch.tensor([1e-8]).to(w_q.device)
            k = w.view(w.shape[0], -1).std(dim=-1) / (w_q.view(w_q.shape[0], -1).std(dim=-1) + eps)
            w_q = (w_q - m_q) * k.view(bshape) + m_q
        if bias_corr:
            w_q = w_q - m_q + m_o
        return w_q
