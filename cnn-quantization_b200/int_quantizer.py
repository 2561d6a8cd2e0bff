"""Drop-in ``IntQuantizer`` for the reference's
``pytorch_quantizer/quantization/qtypes/int_quantizer.py`` (same constructor dict, same ``__call__``,
same mutable attributes, same method names), routed to the fused sm_90a kernels in ``libfqb200.so``.

Where the reference runs ~10 elementwise kernels, several reductions, up to 6 transposed copies and O(C)
host synchronisations per hooked tensor, every dispatch target below is ONE kernel launch on the tensor's own
memory (contiguous NCHW or channels-last) and never reads anything back to the host.

Scope (SURVEY.md section 8): on-the-fly statistics, offline statistics (``-sm use``: parameters solved once per layer,
then one apply-only launch), entropy measurement (``-me``, torch and mid-tread grids) and the activation bias
correction (``-bca``).  Outside the path and raising ``NotImplementedError``: KLD thresholds (``-kld``), ``mix`` clipping.
"""
import math

import numpy as np
import torch

from . import _lib as L
from . import int_quantization
from . import ops

__all__ = ["IntQuantizer", "int_quantizer"]


def _laplace_opt_alpha(w):
    """argmin_a 2*exp(-a) + a^2/(3 w^2)  <=>  a*exp(a) = 3 w^2 (Newton on the Lambert-W equation)."""
    c = 3.0 * w * w
    a = c if c < 1.0 else math.log(c)
    a = max(a, 1e-3)
    for _ in range(100):
        e = math.exp(a)
        na = a - (a * e - c) / (e * (a + 1.0))
        if abs(na - a) <= 1e-16 * abs(na):
            a = na
            break
        a = na
    return a


def _build_tables():
    # int_quantizer.py:41-51: omega grid of 5 decades x 20 steps with a leading 0; alpha = optimal Laplace clip
    res = 20
    omega = np.concatenate([np.linspace(lo, hi, res, endpoint=False)
                            for lo, hi in ((0.01, 0.1), (0.1, 1), (1, 10), (10, 100), (100, 1000))])
    alpha = np.array([_laplace_opt_alpha(w) for w in omega])
    return np.concatenate([[0], omega]), np.concatenate([[0], alpha])


omega_table, alpha_table = _build_tables()


def _to_dev(t, device):
    if isinstance(t, torch.Tensor):
        return t.to(device)
    return torch.tensor(t, dtype=torch.float32).to(device)


class IntQuantizer(object):
    """Mirror of the reference class (int_quantizer.py:56-122).  ``params`` keys as in the reference:
    clipping, stats_kind, kld (optional) and pcq_weights, pcq_act, bit_alloc_act, bit_alloc_weight, bcorr_act,
    bcorr_weight, vcorr_weight, bit_alloc_rmode, bit_alloc_prior, bit_alloc_target_act,
    bit_alloc_target_weight, measure_entropy, logger, mtd_quant (required)."""

    def __init__(self, size, params):
        self.num_bits = size
        self.stochastic = False
        self.int_exp = False
        self.enforce_true_zero = True
        self.clipping = params["clipping"] if "clipping" in params else "no"
        self.stats_kind = params["stats_kind"] if "stats_kind" in params else "mean"
        self.kld = params["kld"] if "kld" in params else False
        self.pcq_w = params["pcq_weights"]
        self.pcq_a = params["pcq_act"]
        self.bit_alloc_act = params["bit_alloc_act"]
        self.bit_alloc_weight = params["bit_alloc_weight"]
        self.bcorr_act = params["bcorr_act"]
        self.bcorr_weight = params["bcorr_weight"]
        self.vcorr_weight = params["vcorr_weight"]
        self.bit_alloc_round = params["bit_alloc_rmode"] == "round"
        self.bit_alloc_prior = params["bit_alloc_prior"]
        ta, tw = params["bit_alloc_target_act"], params["bit_alloc_target_weight"]
        self.bit_alloc_target_act = ta if ta is not None else self.num_bits
        self.bit_alloc_target_weight = tw if tw is not None else self.num_bits
        self.measure_entropy = params["measure_entropy"]
        self.logger = params["logger"]
        self.mtd_quant = params["mtd_quant"]
        self.alpha_gaus = {1: 1.24, 2: 1.71, 3: 2.15, 4: 2.55, 5: 2.93, 6: 3.28, 7: 3.61, 8: 3.92}
        self.alpha_gaus_positive = {1: 1.71, 2: 2.15, 3: 2.55, 4: 2.93, 5: 3.28, 6: 3.61, 7: 3.92, 8: 4.2}
        self.alpha_laplace = {0: 1.05, 1: 1.86, 2: 2.83, 3: 3.89, 4: 5.03, 5: 6.2, 6: 7.41, 7: 8.64, 8: 9.89}
        self.alpha_laplace_positive = {0: 1.86, 1: 2.83, 2: 3.89, 3: 5.02, 4: 6.2, 5: 7.41, 6: 8.64, 7: 9.89, 8: 11.16}
        # statistics manager for `-sm use`: a zero-argument callable returning the manager (the reference stores the
        # singleton CLASS here, inference_quantization_manager.py:413,450,464,471; any object with
        # get_tensor_stat(id, stat, kind) works)
        self.sm = None
        self._stat_cache = {}  # offline-statistics parameters are constants of a layer: solved once, kept on the device
        self.force_positive = False
        self.half_range = False
        # extension (default off = reference behaviour): overwrite the input tensor instead of allocating the result.
        # The manager switches it on for activation tags, where the un-quantized tensor is dead after the hook.
        self.inplace = False
        self.last_entropy = None  # 0-d device tensor of the most recent `-me` measurement
        # diagnostics (default off): keep the [groups, 12] statistics / parameter table of the most recent fused launch
        # (columns _lib.STAT_COLUMNS) in ``last_stats`` - what the parity tests compare with the reference's values
        self.export_stats = False
        self.last_stats = None
        self._relu_follows = False
        self._bca = None
        self._residual, self._residual_used = None, False
        self._defer, self._deferred = False, None
        self._pool, self._pooled = None, False

    # ------------------------------------------------------------------------------------------
    # dispatch (int_quantizer.py:92-122)
    # ------------------------------------------------------------------------------------------
    def __call__(self, tensor, id, tag="", stat_id=None, override_att=None, weight_correction=None, bias=None,
                 relu_follows=False, bias_correct=None, residual=None, defer=False, pool=None):
        """Extensions used by this package's manager (all default to the reference behaviour):
        ``bias_correct`` (None = off, else the "ReLU follows" flag of the call site): the activation bias correction of
        Conv2dWithId.forward (`-bca`, inference_quantization_manager.py:180-196) is applied by the quantizer itself - inside
        the given-parameter launch for channels-last tensors;
        ``residual``: the block input a ResNet block adds to this (its last convolution's) quantized output before the
        closing ReLU; where the launch can take it (per-channel quantization of a channels-last tensor with on-the-fly
        statistics) ``max(quantize(x) + residual, 0)`` is computed in the apply phase and the result is tagged
        ``_fq_residual_fused``; otherwise the operand is ignored and the caller adds it itself;
        ``defer``: this tensor is only ever used as the ``residual`` of another call (the shortcut of a down-sampling
        ResNet block): where both launches can do it, only the statistics phases run now (8 instead of 16 B/element); the
        tensor comes back UNQUANTIZED, tagged ``_fq_deferred = (parameter table, bias)``, and the call that takes it as
        ``residual`` quantizes it on the fly in its apply phase.  The caller must finish a deferred tensor itself
        (call again without ``defer``) when that other call did not fuse;
        ``pool=(2, 2)`` / ``(2, 2, "direct")``: a 2x2 / stride-2 max pooling (floor mode, no padding) - or ``(3, 3)``: 3x3 /
        stride 2 / padding 1 on even H and W, the ResNet stem - is the only consumer of the result - directly, or behind a ReLU that this call's ``relu_follows`` lets the caller skip: where the launch can do it
        (per-channel quantization of a channels-last tensor with an even width) the POOLED quantized tensor comes back,
        tagged ``_fq_pooled`` - the leaf is monotone, so pooling first is bit-identical - and the caller skips its pooling;
        ``relu_follows``: the caller will skip the ReLU that follows when the result is tagged ``_fq_nonneg`` - set on
        every result of a positive (half-range / force-positive) range, where offset 0 gives zero point 0 and every value
        is q * scale >= 0; the compiled leaf's empty-range pass-through then returns max(x, 0) (fqb200_desc.relu_passthrough);
        ``weight_correction=(bias_corr, var_corr)``: the per-output-channel mean / variance correction of
        inference_quantization_manager.py:374-391 is applied inside the same launch that quantizes the weight;
        ``bias``: a per-channel vector added to the tensor before anything else inside the kernel (the folded-BN
        convolution bias, so the convolution itself can run bias-free and a whole pass over the activation is saved)."""
        if override_att is not None:
            orig_att = getattr(self, override_att[0])
            setattr(self, override_att[0], override_att[1])
        self._relu_follows = bool(relu_follows) and self._positive()
        self._bca = bias_correct
        self._residual, self._residual_used = residual, False
        self._defer, self._deferred = bool(defer), None
        self._pool, self._pooled = (tuple(pool) if pool is not None else None), False
        try:
            self._unsupported(stat_id)
            if bias is not None and not self._bias_fusable(tensor):
                # what the convolution would have added (in place when the caller gave the tensor up)
                b = bias.view((1, -1) + (1,) * (tensor.dim() - 2))
                tensor = tensor.add_(b) if self.inplace else tensor + b
                bias = None
            if self.clipping != "no":
                if self.mtd_quant:
                    res = self.mid_tread_quantize_activation(tensor, id, bias=bias)
                else:
                    res = self.gemmlowpClippingQuantize(tensor, id, tag, stat_id=stat_id, clip_type=self.clipping, bias=bias)
            elif self.pcq_w:
                if self.mtd_quant:
                    res = self.mid_tread_quantize_weights_per_channel(tensor, id, weight_correction)
                else:
                    res = self.gemmlowpQuantizeWeightsPerChannel(tensor, id, weight_correction=weight_correction)
            elif self._pc_act(tensor):
                if self.mtd_quant:
                    res = self.mid_tread_quantize_activation_per_channel(tensor, id, bias=bias)
                else:
                    res = self.gemmlowpQuantizeActivationPerChannel(tensor, id, tag, stat_id=stat_id, bias=bias)
            else:
                res = self.gemmlowpMinMaxQuantize(tensor, tag, stat_id=stat_id, weight_correction=weight_correction, bias=bias)
        finally:
            if override_att is not None:
                setattr(self, override_att[0], orig_att)
        if self._relu_follows and isinstance(res, torch.Tensor):
            res._fq_nonneg = res._version   # void as soon as somebody modifies the tensor in place
        if self._residual_used:
            res._fq_residual_fused = True
            res._fq_nonneg = res._version   # the fused epilogue ends with the ReLU
        if self._deferred is not None:
            res._fq_deferred = self._deferred
        if self._pooled:
            res._fq_pooled = self._pooled   # 2 / 3: which pooling the launch has done
        self._defer, self._deferred = False, None
        self._pool, self._pooled = None, False
        self._relu_follows = False
        self._bca = None
        self._residual, self._residual_used = None, False
        return res

    def __repr__(self):
        return ("IntQuantizer - [bits: {}, clipping: {}, bit_alloc_act: {}, bit_alloc_weight: {}, bit_alloc_round: {}, "
                "pcq_w: {}, pcq_a: {}, bcorr_act: {}, bcorr_weight: {}, vcorr_weight: {}, kind: {}]").format(
            self.num_bits, self.clipping, self.bit_alloc_act, self.bit_alloc_weight, self.bit_alloc_round, self.pcq_w,
            self.pcq_a, self.bcorr_act, self.bcorr_weight, self.vcorr_weight, self.stats_kind)

    # ------------------------------------------------------------------------------------------
    # helpers
    # ------------------------------------------------------------------------------------------
    def _unsupported(self, stat_id):
        if self.kld:
            raise NotImplementedError("KLD thresholds are outside the hot-path scope (SURVEY.md section 2, #9)")
        if stat_id is not None and self.sm is None:
            raise RuntimeError("stat_id given but no statistics manager is attached to this quantizer (q.sm)")

    def _pc_act(self, tensor):
        return bool(self.pcq_a and len(tensor.shape) > 3 and (tensor.shape[2] > 1 or tensor.shape[3] > 1))

    def _positive(self):
        return bool(self.force_positive or self.half_range)

    def _bias_fusable(self, tensor):
        """Where the kernel can add the convolution bias itself: the per-channel activation layouts (channel = group)
        and the per-tensor / per-sample min-max layouts of 4-D tensors with H*W % 4 == 0 (bias_period = H*W)."""
        if self.kld or self.mtd_quant and not self._pc_act(tensor):
            return False
        if (self.clipping != "no" or not self.pcq_w) and self._pc_act(tensor) and tensor.shape[1] > 1:
            return True
        minmax = self.clipping == "no" and not self.pcq_w and not self._pc_act(tensor)
        if not (minmax and tensor.dim() == 4):
            return False
        if tensor.is_contiguous():
            return (tensor.shape[2] * tensor.shape[3]) % 4 == 0
        return ops.cl_eligible(tensor)   # channels-last: the bias is a per-thread constant (bias_period = -C)

    @staticmethod
    def _dense(tensor):
        return tensor.is_contiguous() or (tensor.dim() == 4 and tensor.is_contiguous(memory_format=torch.channels_last))

    def _out(self, tensor):
        return tensor if (self.inplace and self._dense(tensor)) else None

    @staticmethod
    def _channels_last(tensor):
        """An NCHW-shaped activation stored NHWC that the channels-last kernels take as is: C % 4 == 0, C <= 2048 (else it
        is made NCHW-contiguous first, like every other strided input)."""
        return ops.cl_eligible(tensor)

    # `-me` (SURVEY.md 8f rank 3): the apply phase histograms the integer grid into 256 counters; the Shannon entropy of
    # utils/entropy.py:6-17 (which runs torch.unique over the whole tensor) is a 256-element computation afterwards
    def _hist(self, tensor):
        return torch.zeros(256, dtype=torch.int64, device=tensor.device) if self.measure_entropy else None

    @staticmethod
    def entropy_from_hist(hist):
        p = hist[hist > 0].to(torch.float32)
        p = p / p.sum()
        return -(p * torch.log2(p)).sum()

    def _log_entropy(self, hist, id, meter, numel):
        if hist is None:
            return
        self.last_entropy = self.entropy_from_hist(hist)
        if self.logger is not None:
            self.logger.log_metric(id + ".entropy", self.last_entropy.item(), step="auto", meterId=meter, weight=numel)

    @staticmethod
    def _nchw_layout(tensor):
        n, c = tensor.shape[0], tensor.shape[1]
        return (n, c, tensor.numel() // (n * c))

    def _range_mode(self, clip_type):
        if clip_type == "laplace":
            return L.RANGE_LAPLACE, 0.0
        if clip_type == "gaus":
            return L.RANGE_GAUS, 0.0
        if "std" in clip_type:
            return L.RANGE_KSTD, float(clip_type.replace("std", ""))
        raise NotImplementedError("clipping %r needs offline statistics or is undefined in the reference" % clip_type)

    def _prior(self):
        return L.PRIOR_STD if self.bit_alloc_prior == "gaus" else L.PRIOR_B

    @staticmethod
    def bias_correction_torch(out, out_q, relu_first):
        """`-bca` with stock torch ops (inference_quantization_manager.py:180-196; reductions over (N, H, W) directly, no
        transposes): the fallback for tensors the fused channels-last launch does not take."""
        if relu_first:
            out = torch.nn.functional.relu(out)
        dims = (0, 2, 3)
        q_bias = out.sum(dims) - out_q.sum(dims)
        count = (out > 0).sum(dims).to(q_bias.dtype)
        q_bias = q_bias / (count + 1e-8)
        out_q += (out_q > 0).to(out_q.dtype) * q_bias.view(1, -1, 1, 1)
        return out_q

    def _quantize1(self, tensor, delta, offset, bits=None, layout=None, bias=None):
        """Mode A launch; with ``bias_correct`` set the activation bias correction rides along."""
        if self._bca is None or tensor.dim() != 4:
            if (self._defer and layout is not None and ops.cl_eligible(tensor, layout) and torch.is_tensor(delta)
                    and delta.numel() == layout[1] and not self.measure_entropy):
                # `defer` with known parameters: nothing to launch at all - the call that takes the tensor as its residual
                # gets the leaf parameters as the table a stats_only launch would have exported (columns 8..11)
                self._deferred = (self._given_table(delta, offset, bits), bias)
                return tensor
            if (layout is not None and (self._residual is not None or self._pool is not None) and ops.cl_eligible(tensor, layout)
                    and torch.is_tensor(delta) and delta.numel() == layout[1] and not self.measure_entropy):
                # the same leaf through the descriptor entry point, which can also finish a ResNet block / pool (`-sm use`)
                return self._launch(tensor, layout, channels_last=True, range_mode=L.RANGE_GIVEN, leaf=L.LEAF_TORCH,
                                    num_bits=min(self.num_bits, 8), given=(delta, offset, bits), bias=bias, out=self._out(tensor))
            return ops.quantize1(tensor, delta, offset, self.num_bits, bits=bits, layout=layout, bias=bias, out=self._out(tensor))
        relu_first = bool(self._bca)
        c = tensor.shape[1]
        if c % 4 == 0 and 4 <= c <= 2048:
            x = tensor if ops.cl_eligible(tensor) else tensor.contiguous(memory_format=torch.channels_last)
            if ops.cl_eligible(x):
                return ops.quantize1_bca(x, delta, offset, self.num_bits, bits=bits, bias=bias, relu_first=relu_first,
                                         out=x if (self.inplace or x is not tensor) else None)
        ref = tensor if bias is None else tensor + bias.view(1, -1, 1, 1)
        return self.bias_correction_torch(ref, ops.quantize1(ref, delta, offset, self.num_bits, bits=bits, layout=layout), relu_first)

    def _given_table(self, delta, offset, bits):
        """[C, 12] parameter table (``_lib.STAT_COLUMNS``) of the torch leaf for given per-channel (delta, offset, bits):
        the arithmetic of int_quantizer.py:557-572 as the kernels do it (make_leaf_param), cached per parameter set."""
        key = ("table", delta.data_ptr(), offset.data_ptr(), None if bits is None else bits.data_ptr(), self.num_bits)
        hit = self._stat_cache.get(key)
        if hit is not None and hit[0] is delta and hit[1] is offset and hit[2] is bits:
            return hit[3]
        b = bits if bits is not None else torch.full_like(delta, float(min(self.num_bits, 8)))
        qmax = torch.pow(2.0, b) - 1.0
        scale = torch.where(qmax > 0, delta / qmax, torch.zeros_like(delta)).clamp_min(1e-8)
        zp = torch.round(0.0 - offset / scale)
        table = torch.zeros((delta.numel(), L.STATS_STRIDE), dtype=torch.float32, device=delta.device)
        table[:, 5], table[:, 6], table[:, 7] = delta, offset, b
        table[:, 8], table[:, 9], table[:, 10], table[:, 11] = scale, zp, qmax, 2.0   # flags: FLAG_TRUE_ZERO
        self._stat_cache[key] = (delta, offset, bits, table)   # the operands are kept alive with the entry
        return table

    def _residual_kw(self, tensor, channels_last, rows=False, bias=None):
        """kwargs of the fused block epilogue when this launch can take it: the channels-last per-channel kernel, or
        (``rows``) the per-sample / per-tensor min-max kernel, which takes any dense order."""
        r = self._residual
        if (r is None or self.measure_entropy or r.shape != tensor.shape or r.stride() != tensor.stride()
                or r.dtype != torch.float32 or r.device != tensor.device):
            return {}
        if rows:
            n = tensor.shape[0]
            dense = tensor.is_contiguous() or (tensor.dim() == 4 and tensor.is_contiguous(memory_format=torch.channels_last))
            if not (dense and tensor.dim() == 4 and n <= 4096 and (tensor.numel() // n) % 4 == 0
                    and tensor.data_ptr() % 16 == 0 and r.data_ptr() % 16 == 0):
                return {}
        elif not channels_last:
            return {}
        kw = dict(residual=r, residual_relu=True)
        deferred = getattr(r, "_fq_deferred", None)
        if deferred is not None:   # the shortcut arrives raw, with its parameter table: quantized in our apply phase
            stats, rbias = deferred
            if (rbias is None) != (bias is None) or (rbias is not None and rbias.numel() != bias.numel()) or self.mtd_quant:
                return {}
            kw.update(residual_stats=stats, residual_bias=rbias)
        self._residual_used = True
        return kw

    def _launch(self, tensor, layout, channels_last=False, rows=False, **kw):
        """One fused launch of the activation paths that can end a ResNet block: deferred (statistics only, see
        ``__call__``), with the block epilogue (``residual``), or plain."""
        if self._defer and kw.get("hist") is None and kw.get("range_mode") != L.RANGE_GIVEN and self._can_defer(tensor, channels_last, rows):
            skw = {k: v for k, v in kw.items() if k not in ("out", "hist")}
            stats = ops.fused(tensor, layout, stats_only=True, channels_last=channels_last, **skw)
            if self.export_stats:
                self.last_stats = stats
            self._deferred = (stats, kw.get("bias"))
            return tensor
        # (a ReLU between quantizer and pooling must be one the caller is going to skip: it has to hand the SAME tensor on)
        if (self._pool is not None and self._pool[:2] in ((2, 2), (3, 3)) and (self._relu_follows or self._pool[2:] == ("direct",))
                and ((channels_last and not rows) or (rows and kw.get("bias") is not None and kw.get("bias_period", 0) < 0
                                                      and tensor.dim() == 4 and not tensor.is_contiguous()
                                                      and tensor.is_contiguous(memory_format=torch.channels_last)
                                                      and tensor.shape[1] % 4 == 0 and tensor.shape[1] <= 2048))
                and kw.get("hist") is None and self._residual is None and not self._defer
                and tensor.dim() == 4 and tensor.shape[2] >= 2 and tensor.shape[3] >= 2 and tensor.shape[3] % 2 == 0
                and (self._pool[0] == 2 or (tensor.shape[2] % 2 == 0 and tensor.shape[1] <= 896))):   # 3x3: 9 * C/4 vectors per stage
            kw.pop("out", None)   # only the pooled tensor is written
            self._pooled = self._pool[0]
            return self._fused(tensor, layout, channels_last=channels_last, pool=self._pool[:2], **kw)
        return self._fused(tensor, layout, channels_last=channels_last, **kw,
                           **self._residual_kw(tensor, channels_last, rows=rows, bias=kw.get("bias")))

    def _can_defer(self, tensor, channels_last, rows):
        if self.measure_entropy or self.mtd_quant or tensor.dim() != 4 or tensor.dtype != torch.float32:
            return False
        if rows:
            n = tensor.shape[0]
            dense = tensor.is_contiguous() or tensor.is_contiguous(memory_format=torch.channels_last)
            return dense and n <= 4096 and (tensor.numel() // n) % 4 == 0 and tensor.data_ptr() % 16 == 0
        return bool(channels_last)

    def _fused(self, tensor, layout, **kw):
        """ops.fused, keeping the exported statistics table when ``export_stats`` is set."""
        if not self.export_stats:
            return ops.fused(tensor, layout, **kw)
        res, self.last_stats = ops.fused(tensor, layout, want_stats=True, **kw)
        return res

    # ------------------------------------------------------------------------------------------
    # offline statistics (`-sm use`): every tensor becomes "mode A" - parameters known up front, one read + one write
    # ------------------------------------------------------------------------------------------
    def _stat(self, stat_id, name, kind="mean"):
        return self.sm().get_tensor_stat(stat_id, name, kind)

    def _cached(self, key, build):
        v = self._stat_cache.get(key)
        if v is None:
            v = self._stat_cache[key] = build()
        return v

    def _stat_bits(self, stat_id, device, target):
        """Per-channel bit widths from the collected prior statistic (int_quantizer.py:236-247, :430-438)."""
        prior = "std" if self.bit_alloc_prior == "gaus" else "b"
        pr = _to_dev(np.asarray(self._stat(stat_id, prior, "mean"), dtype=np.float32), device)
        return self.get_bits_alloc_fixed_target(pr, target, self.bit_alloc_round)

    def _clipping_params_from_stats(self, tensor, stat_id, clip_type):
        """(delta, offset, bits, per_channel) of gemmlowpClippingQuantize in use mode (int_quantizer.py:327-359 with
        :227-300), computed once per (layer, configuration)."""
        positive = self._positive()
        pc_shape = self._pc_act(tensor)
        key = ("clip", stat_id, clip_type, self.num_bits, positive, pc_shape, self.bit_alloc_act, self.bit_alloc_prior,
               self.bit_alloc_round, self.bit_alloc_target_act, str(tensor.device))

        def build():
            dev = tensor.device
            mn, mx, mean = (self._stat(stat_id, k, "mean") for k in ("min", "max", "mean"))
            per_channel = pc_shape and np.size(mn) > 1 and np.size(mx) > 1
            table_l = self.alpha_laplace_positive if positive else self.alpha_laplace
            table_g = self.alpha_gaus_positive if positive else self.alpha_gaus
            bits = None
            if clip_type == "laplace":
                b = self._stat(stat_id, "b", "mean")
                if self.bit_alloc_act and per_channel and self.num_bits <= 4:
                    bits = self._stat_bits(stat_id, dev, self.bit_alloc_target_act)
                    factor = torch.tensor(np.array([table_l[int(v)] for v in bits.tolist()]), dtype=torch.float32, device=dev)
                else:
                    factor = table_l[self.num_bits]
                alpha = _to_dev(np.asarray(b, dtype=np.float32) if per_channel else b, dev) * factor
            elif clip_type == "gaus":
                alpha = self._stat(stat_id, "std", "mean") * table_g[self.num_bits]
            elif "std" in clip_type:
                alpha = float(clip_type.replace("std", "")) * self._stat(stat_id, "std", "mean")
            else:
                raise NotImplementedError("clipping %r is not supported with offline statistics" % clip_type)
            if per_channel:
                rng, off = self.alpha2DeltaOffset(alpha if isinstance(alpha, torch.Tensor) else np.asarray(alpha, dtype=np.float32),
                                                  np.asarray(mx, dtype=np.float32), np.asarray(mn, dtype=np.float32),
                                                  np.asarray(mean, dtype=np.float32))
                off_t = _to_dev(off, dev)
                rng_t = _to_dev(rng, dev)
                max_t = off_t + rng_t                      # :351
                c = tensor.shape[1]
                off_t = off_t.reshape(-1).expand(c) if off_t.numel() == 1 else off_t.reshape(-1)
                if self.bit_alloc_act and self.num_bits <= 4 and bits is None:
                    bits = self._stat_bits(stat_id, dev, self.bit_alloc_target_act)
                return (max_t.reshape(-1) - off_t).contiguous(), off_t.contiguous(), bits, True
            alpha_f = float(alpha)
            rng, off = self.alpha2DeltaOffset(alpha_f, float(mx), float(mn), float(mean))
            return (torch.tensor(rng, dtype=torch.float32, device=dev), torch.tensor(off, dtype=torch.float32, device=dev),
                    None, False)

        return self._cached(key, build)

    # ------------------------------------------------------------------------------------------
    # dispatch targets
    # ------------------------------------------------------------------------------------------
    def gemmlowpClippingQuantize(self, tensor, id, tag="", stat_id=None, clip_type="laplace", bias=None):
        """ACIQ clipping, int_quantizer.py:327-359: per channel (pcq_a, 4-D, HW>1, C>1; fp32 parameter math,
        optional bit allocation) or per tensor (float64 parameter math)."""
        self._unsupported(stat_id)
        if stat_id is not None:
            delta, offset, bits, per_channel = self._clipping_params_from_stats(tensor, stat_id, clip_type)
            if per_channel:
                return self._quantize1(tensor, delta, offset, bits=bits, layout=self._nchw_layout(tensor), bias=bias)
            if self._bca is not None and tensor.dim() == 4:
                return self._quantize1(tensor, delta, offset, bias=bias)   # one parameter set, per-channel correction
            if bias is not None:
                tensor = tensor.add_(bias.view(1, -1, 1, 1)) if self.inplace else tensor + bias.view(1, -1, 1, 1)
            return ops.quantize1(tensor, delta, offset, self.num_bits, out=self._out(tensor))
        mode, k = self._range_mode(clip_type)
        if self._pc_act(tensor) and tensor.shape[1] > 1:
            hist = self._hist(tensor)  # the reference measures entropy in gemmlowpQuantizeActivationPerChannel (:442-445)
            res = self._launch(tensor, self._nchw_layout(tensor), channels_last=self._channels_last(tensor),
                               scope=L.SCOPE_GROUP, range_mode=mode, clip_k=k,
                               leaf=L.LEAF_TORCH, num_bits=self.num_bits, positive=self._positive(),
                               bit_alloc=self.bit_alloc_act, bit_alloc_prior=self._prior(),
                               bit_alloc_round=self.bit_alloc_round, bit_alloc_target=self.bit_alloc_target_act,
                               bias=bias, out=self._out(tensor), hist=hist)
            self._log_entropy(hist, id, "avg.entropy.act", tensor.numel())
            return res
        return self._fused(tensor, (1, 1, tensor.numel()), scope=L.SCOPE_GROUP, range_mode=mode, clip_k=k,
                         leaf=L.LEAF_TORCH, num_bits=self.num_bits, positive=self._positive(), solve_f64=True,
                         out=self._out(tensor), any_dense_format=True)

    def gemmlowpMinMaxQuantize(self, tensor, tag="", stat_id=None, weight_correction=None, bias=None):
        """Per-tensor min/max range through the compiled-leaf arithmetic, int_quantizer.py:361-379 + :605-614.
        Activations (tag contains 'activation', not 'classifier') use the batch average of per-sample min/max."""
        self._unsupported(stat_id)
        if bias is not None and stat_id is not None:
            tensor = tensor.add_(bias.view(1, -1, 1, 1)) if self.inplace else tensor + bias.view(1, -1, 1, 1)
            bias = None
        if stat_id is not None:
            # int_quantizer.py:362-369: collected min/max ('mean' kind, or min-of-min / max-of-max), compiled leaf
            kmin, kmax = ("mean", "mean") if self.stats_kind == "mean" else ("min", "max")
            min_ = float(self._stat(stat_id, "min", kmin))
            max_ = float(self._stat(stat_id, "max", kmax))
            if self._positive():
                min_ = 0.0
            delta = np.float32(max_) - np.float32(min_)
            preserve_zero = bool((np.float32(min_) + delta) > 0 and min_ < 0)
            if delta > 0:
                if self._bca is not None and tensor.dim() == 4:
                    return self.bias_correction_torch(tensor, ops.float2gemmlowp(tensor, float(delta), min_, self.num_bits,
                                                                                 self.int_exp, preserve_zero, None), bool(self._bca))
                return ops.float2gemmlowp(tensor, float(delta), min_, self.num_bits, self.int_exp, preserve_zero, None,
                                          out=self._out(tensor))
            return torch.relu_(tensor) if (self._relu_follows and self.inplace) else (torch.relu(tensor) if self._relu_follows else tensor)
        avg = ("activation" in tag and "classifier" not in tag)
        kw = dict(range_mode=L.RANGE_MINMAX, leaf=L.LEAF_COMPILED, num_bits=self.num_bits, positive=self._positive(),
                  relu_passthrough=self._relu_follows)
        bias_cl = bias is not None and not tensor.is_contiguous()
        if bias is not None:
            kw.update(bias=bias, bias_period=-tensor.shape[1] if bias_cl else tensor.shape[2] * tensor.shape[3])
        if weight_correction is not None and any(weight_correction):
            rows = tensor.shape[0]
            return self._fused(tensor, (1, rows, tensor.numel() // rows), scope=L.SCOPE_TENSOR,
                             bias_corr=weight_correction[0], var_corr=weight_correction[1], **kw)
        n = tensor.shape[0]
        # min / max and a scalar apply do not care about the order inside a sample; a channels-last bias indexes that order
        # (these are the launches of the row kernel, which can also take the block's residual)
        kw["any_dense_format"] = bias is None or bias_cl
        if avg:
            return self._launch(tensor, (1, n, tensor.numel() // n), rows=kw["any_dense_format"], scope=L.SCOPE_GROUP_MEAN,
                                out=self._out(tensor), **kw)
        if bias is not None:
            # rows = samples so that the channel of an element is its column / (H*W); the global min / max is the
            # min / max of the per-row ones (scope TENSOR): identical to the flat per-tensor reduction
            return self._launch(tensor, (1, n, tensor.numel() // n), rows=kw["any_dense_format"], scope=L.SCOPE_TENSOR,
                                out=self._out(tensor), **kw)
        return self._fused(tensor, (1, 1, tensor.numel()), scope=L.SCOPE_GROUP, out=self._out(tensor), **kw)

    def gemmlowpQuantizeActivationPerChannel(self, tensor, id, tag="", stat_id=None, min_=None, max_=None, bias=None):
        """Per-channel min/max (0 lower bound when positive) with optional bit allocation, int_quantizer.py:409-451."""
        self._unsupported(stat_id)
        layout = self._nchw_layout(tensor)
        if stat_id is not None and min_ is None and max_ is None:
            key = ("pc", stat_id, self.num_bits, self._positive(), self.stats_kind, self.bit_alloc_act, self.bit_alloc_prior,
                   self.bit_alloc_round, self.bit_alloc_target_act, str(tensor.device))

            def build():
                dev, c = tensor.device, layout[1]
                mn = torch.zeros(c, device=dev) if self._positive() else _to_dev(
                    np.asarray(self._stat(stat_id, "min", self.stats_kind), dtype=np.float32), dev).reshape(-1)
                mx = _to_dev(np.asarray(self._stat(stat_id, "max", self.stats_kind), dtype=np.float32), dev).reshape(-1)
                bits = self._stat_bits(stat_id, dev, self.bit_alloc_target_act) if (self.bit_alloc_act and self.num_bits <= 4) else None
                return (mx - mn).contiguous(), mn.contiguous(), bits

            delta, offset, bits = self._cached(key, build)
            return self._quantize1(tensor, delta, offset, bits=bits, layout=layout, bias=bias)
        if min_ is None and max_ is None:
            hist = self._hist(tensor)
            res = self._launch(tensor, layout, channels_last=self._channels_last(tensor),
                               scope=L.SCOPE_GROUP, range_mode=L.RANGE_MINMAX, leaf=L.LEAF_TORCH,
                               num_bits=self.num_bits, positive=self._positive(), bit_alloc=self.bit_alloc_act,
                               bit_alloc_prior=self._prior(), bit_alloc_round=self.bit_alloc_round,
                               bit_alloc_target=self.bit_alloc_target_act, bias=bias, out=self._out(tensor), hist=hist)
            self._log_entropy(hist, id, "avg.entropy.act", tensor.numel())
            return res
        if bias is not None:
            tensor = tensor + bias.view(1, -1, 1, 1)
        # explicit bounds (API compatibility): statistics pass for what is missing, then the given-parameter leaf
        st = ops.fused(tensor, layout, num_bits=min(self.num_bits, 8), bit_alloc=self.bit_alloc_act,
                       bit_alloc_prior=self._prior(), bit_alloc_round=self.bit_alloc_round,
                       bit_alloc_target=self.bit_alloc_target_act, stats_only=True)
        c = layout[1]
        if min_ is None:
            min_ = torch.zeros(c, device=tensor.device) if self._positive() else st[:, 0]
        if max_ is None:
            max_ = st[:, 1]
        min_ = _to_dev(min_, tensor.device).reshape(-1)
        max_ = _to_dev(max_, tensor.device).reshape(-1)
        if min_.numel() == 1:
            min_ = min_.expand(c)
        if max_.numel() == 1:
            max_ = max_.expand(c)
        bits = st[:, 7].contiguous() if (self.bit_alloc_act and self.num_bits <= 4) else None
        return ops.quantize1(tensor, (max_ - min_).contiguous(), min_.contiguous(), self.num_bits, bits=bits,
                             layout=layout)

    def gemmlowpQuantizeWeightsPerChannel(self, tensor, id, min_=None, max_=None, weight_correction=None):
        """Per-output-channel min/max with optional bit allocation from the row std, int_quantizer.py:453-476."""
        rows = tensor.shape[0]
        layout = (1, rows, tensor.numel() // rows)
        if min_ is not None or max_ is not None:
            t = tensor.reshape(rows, -1)
            mn = _to_dev(min_, tensor.device) if min_ is not None else t.min(-1)[0]
            mx = _to_dev(max_, tensor.device) if max_ is not None else t.max(-1)[0]
            bits = None
            if self.bit_alloc_weight and self.num_bits <= 4:
                bits = self.get_bits_alloc_fixed_target(t.std(-1), self.bit_alloc_target_weight, self.bit_alloc_round)
            return ops.quantize1(tensor, mx - mn, mn, self.num_bits, bits=bits, layout=layout)
        bc, vc = weight_correction if weight_correction is not None else (False, False)
        hist = self._hist(tensor)
        res = self._fused(tensor, layout, scope=L.SCOPE_GROUP, range_mode=L.RANGE_MINMAX, leaf=L.LEAF_TORCH,
                        num_bits=self.num_bits, positive=False, bit_alloc=self.bit_alloc_weight,
                        bit_alloc_prior=L.PRIOR_STD, bit_alloc_round=self.bit_alloc_round,
                        bit_alloc_target=self.bit_alloc_target_weight, bias_corr=bc, var_corr=vc, hist=hist)
        self._log_entropy(hist, id, "avg.entropy.weight", tensor.numel())
        return res

    # mid-tread "bin allocation" quantizer, int_quantizer.py:147-225
    # `-me` on the mid-tread grid (int_quantizer.py:216-221): the grid is signed, clamped to per-channel and generally
    # FRACTIONAL bounds c_min / c_max, and the reference runs torch.unique over the float grid of all channels together -
    # so every channel's clamp bounds are symbols of their own.  The channels-last kernel histograms the integers and
    # counts the elements sitting on a bound per channel; the symbol table is assembled from those (a few thousand entries).
    MT_HIST_BINS, MT_HIST_OFFSET = 8192, 4096

    @staticmethod
    def mid_tread_entropy_from_hist(hist, offset, clamped, c_min, c_max):
        dev = hist.device
        values = torch.cat([torch.arange(hist.numel(), device=dev, dtype=torch.float32) - float(offset),
                            c_min.reshape(-1).float(), c_max.reshape(-1).float()])
        counts = torch.cat([hist.double(), clamped[:, 0].double(), clamped[:, 1].double()])
        keep = counts > 0
        values, counts = values[keep], counts[keep]
        _, inv = torch.unique(values, return_inverse=True)           # equal floats are ONE symbol, as for torch.unique
        merged = torch.zeros(int(inv.max()) + 1 if inv.numel() else 0, dtype=torch.float64, device=dev).scatter_add_(0, inv, counts)
        p = (merged / merged.sum()).float()
        return -(p * torch.log2(p)).sum()

    def _mid_tread_entropy_torch(self, rows2d, target, clip, sym):
        """The same measurement with stock torch ops on a [R, K] view (weights, non-channels-last activations: small or
        rare tensors; the arithmetic follows int_quantizer.py:185-221 step by step)."""
        t = rows2d
        omega = self.get_omega(t.std(-1), target_bins=(2 ** target)).round()
        if clip:
            am = t.new_tensor(self.get_alpha_mult(omega, sym=sym))
            mu = t.mean(dim=-1)
            b = torch.mean(torch.abs(t - mu.unsqueeze(-1)), dim=-1)
            rng = (2 * am * b) if sym else (torch.max(mu, mu.new_tensor([0.])) + am * b)
        else:
            rng = (t.max(-1)[0] - t.min(-1)[0]) if sym else t.max(-1)[0]
        step = torch.where(omega > 0, rng / omega, t.new_tensor([np.finfo(np.float32).max]))
        grid = (t / step.unsqueeze(-1)).round_()
        if clip:
            mu_q = mu / step if sym else torch.max(mu, mu.new_tensor([0.])) / step
            c_max = mu_q + (omega / 2 if sym else omega)
            c_min = (mu_q - omega / 2) if sym else t.new_tensor([0])
            grid = torch.max(torch.min(grid, c_max.unsqueeze(-1)), c_min.unsqueeze(-1))
        counts = torch.unique(grid.flatten(), return_counts=True)[1].float()
        p = counts / counts.sum()
        return -(p * torch.log2(p)).sum()

    def _log_mt_entropy(self, entropy, id, meter, numel):
        self.last_entropy = entropy
        if self.logger is not None:
            self.logger.log_metric(id + ".entropy", entropy.item(), step="auto", meterId=meter, weight=numel)

    def mid_tread_quantize_weights_per_channel(self, tensor, id, weight_correction=None):
        rows = tensor.shape[0]
        bc, vc = weight_correction if weight_correction is not None else (False, False)
        if self.measure_entropy:
            self._log_mt_entropy(self._mid_tread_entropy_torch(tensor.reshape(rows, -1), self.bit_alloc_target_weight, False, True),
                                 id, "avg.entropy.weight", tensor.numel())
        return self._fused(tensor, (1, rows, tensor.numel() // rows), leaf=L.LEAF_MIDTREAD, positive=False,
                         mt_target=self.bit_alloc_target_weight, mt_clip=False, bias_corr=bc, var_corr=vc)

    def mid_tread_quantize_activation(self, tensor, id, bias=None):
        if self._pc_act(tensor):
            return self.mid_tread_quantize_activation_per_channel(tensor, id, bias=bias)
        if bias is not None:
            tensor = tensor + bias.view((1, -1) + (1,) * (tensor.dim() - 2))
        return self._fused(tensor, (1, 1, tensor.numel()), leaf=L.LEAF_MIDTREAD, positive=self._positive(),
                         mt_target=self.bit_alloc_target_act, mt_clip=True, out=self._out(tensor))

    def mid_tread_quantize_activation_per_channel(self, tensor, id, bias=None):
        layout = self._nchw_layout(tensor)
        kw = dict(leaf=L.LEAF_MIDTREAD, positive=self._positive(), mt_target=self.bit_alloc_target_act, mt_clip=True, bias=bias,
                  out=self._out(tensor), channels_last=self._channels_last(tensor))
        if not self.measure_entropy:
            return self._launch(tensor, layout, **kw)   # the mid-tread leaf is monotone too: block epilogue / pooling apply
        if kw["channels_last"]:
            hist = torch.zeros(self.MT_HIST_BINS, dtype=torch.int64, device=tensor.device)
            clamped = torch.zeros((layout[1], 2), dtype=torch.int64, device=tensor.device)
            res, st = ops.fused(tensor, layout, want_stats=True, hist=hist, hist_offset=self.MT_HIST_OFFSET, hist_clamped=clamped, **kw)
            self.last_stats = st
            entropy = self.mid_tread_entropy_from_hist(hist, self.MT_HIST_OFFSET, clamped, st[:, 9], st[:, 10])
        else:
            x = tensor if bias is None else tensor + bias.view(1, -1, 1, 1)
            entropy = self._mid_tread_entropy_torch(x.transpose(0, 1).reshape(layout[1], -1), self.bit_alloc_target_act, True,
                                                    not self._positive())
            res = self._fused(tensor, layout, **kw)
        self._log_mt_entropy(entropy, id, "avg.entropy.act", tensor.numel())
        return res

    def mid_tread_quantization(self, tensor, id, target, clip=False, sym=True):
        """[R, K] view, int_quantizer.py:185-225.  Returns (quantized, None) like the reference without entropy."""
        out = self._fused(tensor, (1, tensor.shape[0], tensor.numel() // tensor.shape[0]), leaf=L.LEAF_MIDTREAD,
                        positive=not sym, mt_target=target, mt_clip=clip)
        return out, None

    # ------------------------------------------------------------------------------------------
    # leaves with caller-provided parameters
    # ------------------------------------------------------------------------------------------
    def __gemmlowpQuantize1__(self, tensor, delta, offset, bit_alloc=None, measure_entropy=False):
        """int_quantizer.py:557-603: [R, K] tensor with [R] parameters, or any shape with 0-d parameters."""
        if measure_entropy:
            out, grid = ops.quantize1(tensor, delta, offset, self.num_bits, bits=bit_alloc, want_grid=True)
            hist = torch.bincount(grid.flatten().to(torch.int64).clamp_(0, 255), minlength=256)
            return out, self.entropy_from_hist(hist)
        return ops.quantize1(tensor, delta, offset, self.num_bits, bits=bit_alloc)

    def __gemmlowpQuantize__(self, tensor, delta, offset):
        """int_quantizer.py:605-614.  Tensor arguments are converted to python floats exactly as the reference's
        pybind call does (a host synchronisation); the dispatch targets above never come through here."""
        preserve_zero = bool(self.enforce_true_zero and (offset + delta) > 0 and offset < 0)
        return int_quantization.float2gemmlowp(tensor.contiguous(), float(delta), float(offset), self.num_bits,
                                               self.int_exp, preserve_zero, None)

    # ------------------------------------------------------------------------------------------
    # statistics / parameter helpers kept for API compatibility (small torch ops on [C]-sized tensors)
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _stats_cols(tensor, layout):
        return ops.fused(tensor, layout, stats_only=True)

    @staticmethod
    def __act_stats__(tensor, stats, avg_over_batch=False):
        """int_quantizer.py:507-528 through one statistics-only launch."""
        cols = {"min": 0, "max": 1, "mean": 2, "b": 3, "std": 4}
        if avg_over_batch:
            n = tensor.shape[0]
            st = IntQuantizer._stats_cols(tensor, (1, n, tensor.numel() // n))
            return {s: st[:, cols[s]].mean(dim=0) for s in stats}
        st = IntQuantizer._stats_cols(tensor, (1, 1, tensor.numel()))
        return {s: st[0, cols[s]] for s in stats}

    @staticmethod
    def __act_stats_perchannel__(tensor, stats, avg_over_batch=False):
        """int_quantizer.py:530-555 without the transposed copy."""
        cols = {"min": 0, "max": 1, "mean": 2, "b": 3, "std": 4}
        n, c = tensor.shape[0], tensor.shape[1]
        hw = tensor.numel() // (n * c)
        if avg_over_batch:
            st = IntQuantizer._stats_cols(tensor, (1, n * c, hw)).view(n, c, -1)
            return {s: st[:, :, cols[s]].mean(dim=0) for s in stats}
        st = IntQuantizer._stats_cols(tensor, (n, c, hw))
        return {s: st[:, cols[s]].contiguous() for s in stats}

    @staticmethod
    def get_bits_alloc(alpha, num_bits, round=False):
        """int_quantizer.py:381-391."""
        budget = len(alpha) * 2 ** num_bits
        p = alpha ** (2.0 / 3)
        bins = (budget * p) / p.sum()
        bits = torch.round(torch.log2(bins)) if round else torch.ceil(torch.log2(bins))
        return bits.clamp_(0, 8)

    @staticmethod
    def get_bits_alloc_fixed_target(alpha, num_bits, round=False):
        """int_quantizer.py:393-407."""
        goal = num_bits
        m = goal
        half_gap = 1.0
        it = 0
        bits = None
        while abs(2 * half_gap) > 0.01 and it < 10:
            it += 1
            bits = IntQuantizer.get_bits_alloc(alpha, num_bits=m, round=round)
            half_gap = (goal - bits.mean()) / 2
            m += half_gap.item()
        return bits

    @staticmethod
    def get_omega(sigma, target_bins):
        """int_quantizer.py:128-135."""
        p = sigma ** (2.0 / 3)
        return (len(sigma) * target_bins * p) / p.sum()

    @staticmethod
    def get_alpha_mult(omega, sym=True):
        """int_quantizer.py:137-145 (the caller's omega is left untouched, as on CUDA tensors in the reference)."""
        om = omega.detach().cpu().numpy().astype(np.float64)
        if not sym:
            om = om * 2
        i = np.minimum(omega_table.searchsorted(om), len(omega_table) - 1)
        inc = (alpha_table[i] - alpha_table[i - 1]) / (omega_table[i] - omega_table[i - 1])
        return alpha_table[i] - inc * (omega_table[i] - om)

    def get_alpha_laplace(self, tensor, stat_id=None, kind="mean", per_channel=False):
        """int_quantizer.py:227-253."""
        self._unsupported(stat_id)
        stats = self.__act_stats_perchannel__ if per_channel else self.__act_stats__
        b = stats(tensor, ["b"])["b"]
        table = self.alpha_laplace_positive if self._positive() else self.alpha_laplace
        if self.bit_alloc_act and per_channel and self.num_bits <= 4:
            prior = "std" if self.bit_alloc_prior == "gaus" else "b"
            pr = stats(tensor, [prior])[prior]
            bits = self.get_bits_alloc_fixed_target(pr, self.bit_alloc_target_act, self.bit_alloc_round)
            factor = torch.tensor([table[int(v)] for v in bits.tolist()], dtype=torch.float32, device=tensor.device)
            return b * factor
        return b * table[self.num_bits]

    def get_alpha_gaus(self, tensor, tag, stat_id=None, per_channel=False):
        """int_quantizer.py:255-264."""
        self._unsupported(stat_id)
        stats = self.__act_stats_perchannel__ if per_channel else self.__act_stats__
        std = stats(tensor, ["std"])["std"]
        return std * (self.alpha_gaus_positive if self._positive() else self.alpha_gaus)[self.num_bits]

    def get_alpha_pstd(self, tensor, p, tag, stat_id=None, per_channel=False):
        """int_quantizer.py:266-275."""
        self._unsupported(stat_id)
        stats = self.__act_stats_perchannel__ if per_channel else self.__act_stats__
        return p * stats(tensor, ["std"])["std"]

    def get_alpha(self, tensor, tag="", stat_id=None, clip_type="laplace", per_channel=False):
        """int_quantizer.py:302-325."""
        if clip_type == "laplace":
            return self.get_alpha_laplace(tensor, stat_id, per_channel=per_channel)
        if clip_type == "gaus":
            return self.get_alpha_gaus(tensor, tag, stat_id, per_channel=per_channel)
        if "std" in clip_type:
            return self.get_alpha_pstd(tensor, float(clip_type.replace("std", "")), tag, stat_id, per_channel=per_channel)
        raise NotImplementedError("clipping %r needs offline statistics" % clip_type)

    def alpha2DeltaOffset(self, alpha, max_value, min_value, mean, clip2max=False):
        """int_quantizer.py:284-300 (numpy arithmetic, host side)."""
        def _np(v):
            return v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v
        alpha, max_value, min_value, mean = map(_np, (alpha, max_value, min_value, mean))
        if self._positive():
            delta = np.maximum(np.array(mean), 0) + alpha
            if clip2max:
                delta = np.minimum(delta, max_value)
            return delta, 0
        delta = 2 * alpha
        if clip2max:
            delta = np.minimum(delta, max_value - min_value)
        return delta, np.maximum(min_value, mean - alpha)


def int_quantizer(qtype, quant_params):
    """Factory with the reference's naming rule (int_quantizer.py:626-632): 'intN' -> N bits."""
    size = int(qtype[len("int"):]) if len(qtype) > len("int") else 32
    return IntQuantizer(size, quant_params)
