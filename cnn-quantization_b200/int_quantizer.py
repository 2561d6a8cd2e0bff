"""Drop-in ``IntQuantizer`` for the reference's
``pytorch_quantizer/quantization/qtypes/int_quantizer.py`` (same constructor dict, same ``__call__``,
same mutable attributes, same method names), routed to the fused sm_90a kernels in ``libfqb200.so``.

Where the reference runs ~10 elementwise kernels, several reductions, up to 6 transposed copies and O(C)
host synchronisations per hooked tensor, every dispatch target below is ONE kernel launch on the tensor's own
memory (contiguous NCHW or channels-last) and never reads anything back to the host.

Scope (SURVEY.md section 8): on-the-fly statistics, offline statistics (``-sm use``: parameters solved once per layer,
then one apply-only launch), KLD thresholds (``-kld``: collected per sample by ops.kld_threshold, applied in use mode as
one apply-only launch of the compiled leaf), entropy measurement (``-me``, torch and mid-tread grids) and the activation
bias correction (``-bca``) and ``mix`` clipping (``-sm use`` only: the per-layer or per-channel choice between no clipping,
Gauss and Laplace by the mse_* statistics collected with ``collect_err``, then one apply-only launch).
"""
import collections
import math

import numpy as np
import torch

from . import _lib as L
from . import int_quantization
from . import ops
from .statistics import refuse_bap_mse

__all__ = ["IntQuantizer", "int_quantizer", "MseCandidates", "WeightMse", "best_candidates", "refuse_clip_weight"]


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

# ACIQ clipping factors per bit width (int_quantizer.py:74-77)
ALPHA_GAUS = {1: 1.24, 2: 1.71, 3: 2.15, 4: 2.55, 5: 2.93, 6: 3.28, 7: 3.61, 8: 3.92}
ALPHA_GAUS_POSITIVE = {1: 1.71, 2: 2.15, 3: 2.55, 4: 2.93, 5: 3.28, 6: 3.61, 7: 3.92, 8: 4.2}
ALPHA_LAPLACE = {0: 1.05, 1: 1.86, 2: 2.83, 3: 3.89, 4: 5.03, 5: 6.2, 6: 7.41, 7: 8.64, 8: 9.89}
ALPHA_LAPLACE_POSITIVE = {0: 1.86, 1: 2.83, 2: 3.89, 3: 5.02, 4: 6.2, 5: 7.41, 6: 8.64, 7: 9.89, 8: 11.16}


def _to_dev(t, device):
    if isinstance(t, torch.Tensor):
        return t.to(device)
    return torch.tensor(t, dtype=torch.float32).to(device)


def refuse_clip_weight(clip_weight="mse", per_channel=True, mid_tread=False, bounds=False, qweight="int8", native=True):
    """Raise where `clip_weight="mse"` cannot run: an unknown value or per-tensor weights (ValueError); the mid-tread
    (-mtq) bins, explicit min_ / max_ bounds, float weights (qweight f32) or a foreign quantizer (NotImplementedError)."""
    if clip_weight not in ("no", "mse"):
        raise ValueError("clip_weight must be 'no' or 'mse', got %r" % (clip_weight,))
    if clip_weight == "no":
        return
    if not per_channel:
        raise ValueError("clip_weight='mse' picks a clipping value per output channel: it needs per_channel_quant_weights")
    if mid_tread:
        raise NotImplementedError("clip_weight='mse' clips the min/max weight quantizer, not the mid-tread (-mtq) bins")
    if bounds:
        raise NotImplementedError("clip_weight='mse' measures each row's own range: explicit min_ / max_ bounds are not "
                                  "supported")
    if qweight == "f32":
        raise NotImplementedError("clip_weight='mse' clips quantized weights, and qweight f32 leaves them in float")
    if not native:
        raise NotImplementedError("clip_weight='mse' runs on this package's CUDA quantizers only")


def best_candidates(err):
    """(column, error) of the least error per row of ``err`` [G, W, 1 + M] (per channel and width: column 0 the min/max
    range, then the M clipping values): the first minimum in column order, so min/max wins exact ties and then the
    earlier multiplier; NaN never wins (statistics.best_columns' rule; a row of NaN keeps min/max)."""
    pick = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err).argmin(2)
    return pick, err.gather(2, pick.unsqueeze(2)).squeeze(2)


class MseCandidates(object):
    """The clipping candidates of measured clipping, shared by one model's quantizers: the float32 multipliers and their
    prior ("laplace": alpha = m * b, "gaus": m * std), with one device copy per device."""

    def __init__(self, multipliers, prior):
        self.multipliers = np.asarray(multipliers, dtype=np.float32).reshape(-1)
        self.prior = prior
        self._mult = {}

    def mult(self, dev):
        m = self._mult.get(dev)
        if m is None:   # pinned and asynchronous: no host synchronisation inside quantize_model or a forward
            m = self._mult[dev] = torch.from_numpy(self.multipliers).pin_memory().to(dev, non_blocking=True)
        return m


class WeightMse(MseCandidates):
    """What `clip_weight="mse"` shares across one model's weight quantizers: the clipping candidates
    (``MseCandidates``), the int32 device flag fqb200_allocate_widths raises on non-finite error tables, and with
    ``report`` (a CSV path) one row of device sums per quantized weight.  Nothing is read back until ``finish``, which
    reads the flag and the report in one copy."""

    REPORT_COLUMNS = ("id", "rows", "bits", "mse_minmax", "mse_chosen", "kept_minmax", "bits_minmax_alloc",
                      "mse_minmax_alloc")

    def __init__(self, multipliers, prior, report=None):
        super(WeightMse, self).__init__(multipliers, prior)
        self.report = report
        self._status = None
        self._rows = []   # (id, rows, numel, float64 device [6]: bits, sse min/max, sse chosen, kept, bits / sse of the
                          # min/max-only allocation)

    def status(self, dev):
        if self._status is None:
            self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        return self._status

    def add(self, id, rows, numel, sums):
        if self.report is not None:
            self._rows.append((id, rows, numel, sums))

    def finish(self):
        """Read the flag and the report sums back (one copy), write the report, and raise ValueError when an allocation
        met a non-finite error."""
        if self._status is None and not self._rows:
            return
        parts = ([self._status.double()] if self._status is not None else []) + [r[3] for r in self._rows]
        host = torch.cat([p.reshape(-1).to(parts[0].device) for p in parts]).cpu().numpy()
        bad = self._status is not None and host[0] != 0
        sums = host[1 if self._status is not None else 0:].reshape(-1, 6)
        rows, self._rows, self._status = self._rows, [], None
        if self.report is not None and rows:
            import csv
            with open(self.report, "w", newline="") as f:
                w = csv.writer(f)
                w.writerow(self.REPORT_COLUMNS)
                for (id, r, n, _), s in zip(rows, sums):
                    w.writerow([id, r, int(s[0]), repr(float(s[1] / n)), repr(float(s[2] / n)), int(s[3]),
                                "" if np.isnan(s[4]) else int(s[4]), "" if np.isnan(s[5]) else repr(float(s[5] / n))])
        if bad:
            raise ValueError("clip_weight='mse': a weight's error table holds NaN or Inf, so its width allocation is not "
                             "defined (bit_alloc.allocate refuses such tables)")


# `-c mse` on the fly without candidates from a manager (a bare quantizer): statistics.MSE_MULTIPLIERS times the Laplace b
_DEFAULT_MSE_CANDIDATES = None


def _default_mse_candidates():
    global _DEFAULT_MSE_CANDIDATES
    if _DEFAULT_MSE_CANDIDATES is None:
        from .statistics import MSE_MULTIPLIERS
        _DEFAULT_MSE_CANDIDATES = MseCandidates(MSE_MULTIPLIERS, "laplace")
    return _DEFAULT_MSE_CANDIDATES


# `-baa -bap mse` on the fly: the width candidates of statistics.bit_candidates per (rule, positive, num_bits), constants
_BIT_CANDIDATES = {}


def _bit_candidates(rule, positive, num_bits):
    key = (rule, bool(positive), num_bits)
    cand = _BIT_CANDIDATES.get(key)
    if cand is None:
        from .statistics import bit_candidates
        cand = _BIT_CANDIDATES[key] = MseCandidates(*bit_candidates(rule, positive, num_bits))
    return cand


# A call site's `-sm use` parameters: per channel, [C] delta / offset and the widths (or None) of the torch leaf; per
# tensor, 0-d delta / offset of the torch leaf (preserve_zero None), or the float range / offset and preserve_zero of the
# compiled leaf, whose range is None where the tensor passes through unquantized.
_UseParams = collections.namedtuple("_UseParams", "per_channel delta offset bits preserve_zero")


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
        self.alpha_gaus = dict(ALPHA_GAUS)
        self.alpha_gaus_positive = dict(ALPHA_GAUS_POSITIVE)
        self.alpha_laplace = dict(ALPHA_LAPLACE)
        self.alpha_laplace_positive = dict(ALPHA_LAPLACE_POSITIVE)
        # statistics manager for `-sm use`: a zero-argument callable returning the manager (the reference stores the
        # singleton CLASS here, inference_quantization_manager.py:413,450,464,471; any object with
        # get_tensor_stat(id, stat, kind) works)
        self.sm = None
        # `-c mse`: the statistics.ClipMseStatistics that reads the collected clipping-MSE curves (set by the manager)
        self.mse_curves = None
        # `-bap mse`: the statistics.BitMseStatistics that reads the collected per-channel error tables (set by the manager)
        self.bit_tables = None
        # `clip_weight="mse"` (set by the manager on its weight quantizers): per output channel the measured best of the
        # min/max range and the clipping candidates of ``weight_mse`` (a WeightMse)
        self.clip_weight = "no"
        self.weight_mse = None
        # `-c mse` on the fly (no statistics manager): the MseCandidates each activation is measured over (set by the
        # manager; None: statistics.MSE_MULTIPLIERS with the Laplace prior)
        self.mse_candidates = None
        # `-baa -bap mse` on the fly (no statistics manager, set by the manager with fly_bits): each per-channel,
        # bit-allocated activation gets the widths that minimise the sum of its own per-channel errors, in every forward
        self.fly_bits = False
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
        self.last_weight_mse = None   # ... and of the most recent `clip_weight="mse"` weight (see _clip_mse_weights)
        self.last_clip_choice = None  # ... and the [groups] chosen columns of the most recent `-c mse` on-the-fly call
        # per-call inputs of ``__call__``'s extensions (reset when the call returns)
        self._relu_follows, self._bca, self._residual, self._defer, self._pool, self._into = False, None, None, False, None, None

    # ------------------------------------------------------------------------------------------
    # dispatch (int_quantizer.py:92-122)
    # ------------------------------------------------------------------------------------------
    def __call__(self, tensor, id, tag="", stat_id=None, override_att=None, weight_correction=None, bias=None,
                 relu_follows=False, bias_correct=None, residual=None, defer=False, pool=None, out=None):
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
        convolution bias, so the convolution itself can run bias-free and a whole pass over the activation is saved);
        ``out``: a channel slice of a wider channels-last tensor (a branch's part of an Inception block's concatenation);
        where the channels-last apply launch, or the per-sample / per-tensor min-max launch of a channels-last tensor with a
        convolution bias, can write it (``ops.slice_eligible``) the result is written there and that
        slice comes back; otherwise the operand is ignored and the caller copies the result itself."""
        if override_att is not None:
            orig_att = getattr(self, override_att[0])
            setattr(self, override_att[0], override_att[1])
        self._relu_follows = bool(relu_follows) and self._positive()
        self._bca = bias_correct
        self._residual = residual
        self._defer = bool(defer)
        self._pool = tuple(pool) if pool is not None else None
        self._into = out
        try:
            self._unsupported(stat_id)
            if bias is not None and not self._bias_fusable(tensor, stat_id):
                # what the convolution would have added (in place when the caller gave the tensor up)
                b = bias.view((1, -1) + (1,) * (tensor.dim() - 2))
                tensor = tensor.add_(b) if self.inplace else tensor + b
                bias = None
            if self.kld:
                res = self.gemmlowpKldQuantize(tensor, tag, stat_id=stat_id)
            elif self.clipping != "no":
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
            if self._relu_follows and isinstance(res, torch.Tensor):
                res._fq_nonneg = res._version   # void as soon as somebody modifies the tensor in place
        finally:
            if override_att is not None:
                setattr(self, override_att[0], orig_att)
            self._relu_follows, self._bca, self._residual, self._defer, self._pool, self._into = False, None, None, False, None, None
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
        if stat_id is not None and self.sm is None:
            raise RuntimeError("stat_id given but no statistics manager is attached to this quantizer (q.sm)")

    def _pc_act(self, tensor):
        return bool(self.pcq_a and len(tensor.shape) > 3 and (tensor.shape[2] > 1 or tensor.shape[3] > 1))

    def _positive(self):
        return bool(self.force_positive or self.half_range)

    def _bias_fusable(self, tensor, stat_id=None):
        """Where the kernel can add the convolution bias itself: the per-channel activation layouts (channel = group)
        and the per-tensor / per-sample min-max layouts of 4-D tensors with H*W % 4 == 0 (bias_period = H*W).  Not `-c mse`
        on the fly: its candidate sums have no bias operand (adding it first is the same single fp32 rounding)."""
        if self.kld or self.mtd_quant and not self._pc_act(tensor):
            return False
        if self.clipping == "mse" and stat_id is None and not self.mtd_quant:
            return False
        if stat_id is None and self._fly_bits_site(tensor):   # the same: its candidate sums have no bias operand
            return False
        if (self.clipping != "no" or not self.pcq_w) and self._pc_act(tensor) and tensor.shape[1] > 1:
            return True
        minmax = self.clipping == "no" and not self.pcq_w and not self._pc_act(tensor)
        if not (minmax and tensor.dim() == 4):
            return False
        if tensor.is_contiguous():
            return (tensor.shape[2] * tensor.shape[3]) % 4 == 0
        return ops.cl_eligible(tensor)   # channels-last: the bias is a per-thread constant (bias_period = -C)

    def _out(self, tensor):
        return tensor if (self.inplace and ops.dense(tensor)) else None

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
        """The prior of the on-the-fly activation launches' bit allocation."""
        if self.bit_alloc_prior == "mse":
            if self.fly_bits and not self._allocates(True):
                return L.PRIOR_B   # above 4 bits nothing is allocated (the launch reads no prior); fly_bits takes the rest
            refuse_bap_mse(needs_use=self.bit_alloc_act)
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

    def _quantize1(self, tensor, delta, offset, bits=None, layout=None, bias=None, table=None):
        """Mode A launch; with ``bias_correct`` set the activation bias correction rides along.  ``table``: the [C, 12]
        parameter table of (delta, offset, bits) when the caller has it (a deferred shortcut hands it on)."""
        if self._bca is None or tensor.dim() != 4:
            # per-channel parameters of a channels-last tensor that the descriptor entry point takes as it is
            if ((self._defer or self._residual is not None or self._pool is not None or self._into is not None) and layout is not None
                    and torch.is_tensor(delta) and delta.numel() == layout[1] and not self.measure_entropy
                    and ops.cl_eligible(tensor, layout)):
                if self._defer:
                    # nothing to launch at all: the call that takes the tensor as its residual gets the leaf parameters as
                    # the table a stats_only launch would have exported (columns 8..11)
                    tensor._fq_deferred = (table if table is not None else self._given_table(delta, offset, bits), bias)
                    return tensor
                # the same leaf through the descriptor entry point, which can also finish a ResNet block / pool (`-sm use`)
                return self._launch(tensor, layout, channels_last=True, range_mode=L.RANGE_GIVEN, leaf=L.LEAF_TORCH,
                                    num_bits=min(self.num_bits, 8), given=(delta, offset, bits), bias=bias, out=self._out(tensor))
            return ops.quantize1(tensor, delta, offset, self.num_bits, bits=bits, layout=layout, bias=bias, out=self._out(tensor))
        relu_first = bool(self._bca)
        if ops.cl_channels_ok(tensor.shape[1]):   # else no channels-last copy would qualify either
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
        if not (ops.rows_eligible(tensor, r) if rows else channels_last):
            return {}
        kw = dict(residual=r, residual_relu=True)
        deferred = getattr(r, "_fq_deferred", None)
        if deferred is not None:   # the shortcut arrives raw, with its parameter table: quantized in our apply phase
            stats, rbias = deferred
            if (rbias is None) != (bias is None) or (rbias is not None and rbias.numel() != bias.numel()) or self.mtd_quant:
                return {}
            kw.update(residual_stats=stats, residual_bias=rbias)
        return kw

    def _launch(self, tensor, layout, channels_last=False, rows=False, **kw):
        """One fused launch of the activation paths that can end a ResNet block: deferred (statistics only, see
        ``__call__``), pooled, with the block epilogue (``residual``), or plain.  Tags the result with what it did."""
        if (self._defer and kw.get("hist") is None and kw.get("range_mode") != L.RANGE_GIVEN and not self.measure_entropy
                and not self.mtd_quant and tensor.dtype == torch.float32 and (ops.rows_eligible(tensor) if rows else channels_last)):
            skw = {k: v for k, v in kw.items() if k not in ("out", "hist")}
            stats = ops.fused(tensor, layout, stats_only=True, channels_last=channels_last, **skw)
            if self.export_stats:
                self.last_stats = stats
            tensor._fq_deferred = (stats, kw.get("bias"))
            return tensor
        # (a ReLU between quantizer and pooling must be one the caller is going to skip: it has to hand the SAME tensor on)
        pool = self._pool
        if pool is not None and (self._relu_follows or pool[2:] == ("direct",)) and not self._defer:
            rows_cl = rows and kw.get("bias_period", 0) < 0 and ops.cl_eligible(tensor)   # C from the channel-fastest bias
            if (ops.pool_request_ok(tensor, pool[:2], channels_last or rows_cl, residual=self._residual, hist=kw.get("hist"))
                    and ops.pool_tile_fits(tensor, pool[0])):
                kw.pop("out", None)   # only the pooled tensor is written
                res = self._fused(tensor, layout, channels_last=channels_last, pool=pool[:2], **kw)
                res._fq_pooled = pool[0]   # 2 / 3: which pooling the launch has done
                return res
        rkw = self._residual_kw(tensor, channels_last, rows=rows, bias=kw.get("bias"))
        # (a rows launch knows C, and so the pixels of a slice, from its channel-fastest bias)
        if not rkw and self._into is not None and ops.slice_eligible(tensor, self._into, channels_last,
                                                                     bias_period=kw.get("bias_period", 0) if rows else 0):
            kw["out"] = self._into
        res = self._fused(tensor, layout, channels_last=channels_last, **kw, **rkw)
        if rkw:
            res._fq_residual_fused = True
            res._fq_nonneg = res._version   # the fused epilogue ends with the ReLU
        return res

    def _fused(self, tensor, layout, **kw):
        """ops.fused, keeping the exported statistics table when ``export_stats`` is set."""
        if not self.export_stats or kw.get("range_mode") == L.RANGE_GIVEN:   # given parameters: nothing to export
            return ops.fused(tensor, layout, **kw)
        res, self.last_stats = ops.fused(tensor, layout, want_stats=True, **kw)
        return res

    # ------------------------------------------------------------------------------------------
    # offline statistics (`-sm use`): every tensor becomes "mode A" - parameters known up front, one read + one write
    # ------------------------------------------------------------------------------------------
    def _stat(self, stat_id, name, kind="mean"):
        return self.sm().get_tensor_stat(stat_id, name, kind)

    def _allocates(self, per_channel):
        """Whether a call site's activation channels get their own widths (int_quantizer.py:236-247, :430-438)."""
        return bool(self.bit_alloc_act and per_channel and self.num_bits <= 4)

    def _fly_bits_site(self, tensor):
        """Whether ``fly_bits`` allocates this activation on the fly: a per-channel (per-channel ACIQ needs C > 1),
        bit-allocated call site of the clipping or min/max dispatch target."""
        return bool(self.fly_bits and not self.kld and not self.mtd_quant and self._pc_act(tensor)
                    and (self.clipping == "no" or tensor.shape[1] > 1) and self._allocates(True))

    def _use_bits(self, stat_id, per_channel, dev):
        """None, or the float32 [C] widths of a per-channel, bit-allocated call site from ``_stat_bits``."""
        return self._stat_bits(stat_id, dev, self.bit_alloc_target_act) if self._allocates(per_channel) else None

    def _stat_bits(self, stat_id, device, target):
        """Per-channel bit widths from the collected prior statistic (int_quantizer.py:236-247, :430-438), or with
        ``bit_alloc_prior="mse"`` the widths bit_alloc.allocate gives the layer's collected error tables."""
        if self.bit_alloc_prior == "mse":
            return self._mse_bits(stat_id, device, target)
        prior = "std" if self.bit_alloc_prior == "gaus" else "b"
        pr = _to_dev(np.asarray(self._stat(stat_id, prior, "mean"), dtype=np.float32), device)
        return self.get_bits_alloc_fixed_target(pr, target, self.bit_alloc_round)

    def _mse_bits(self, stat_id, device, target):
        """`-bap mse`: float32 [C] widths minimising the sum of the layer's measured per-channel errors (bit_mse.pkl,
        collected with collect_bits under this run's clipping rule) for the budget of ``target`` bits per channel."""
        from .bit_alloc import allocate
        refuse_bap_mse(kld=self.kld, clipping=self.clipping, widths_alone=True)
        mse = self._bit_table(stat_id, self.clipping)[0]
        return torch.tensor(allocate(mse, target), dtype=torch.float32, device=device)

    def _bit_table(self, stat_id, rule):
        """(float64 [C, 9] errors of widths 0..8, float32 [C] scale, float32 [C, 9] best multipliers of a joint table
        (``rule`` "mse") or None) of the layer's `-bap mse` table, checked to exist, to be measured under ``rule`` and to
        have a row per channel of the summary scale: b (std for mse_prior "gaus") for a joint table, else max."""
        if self.bit_tables is None:
            raise KeyError("-bap mse needs the per-channel error tables of layer %r: collect them with collect_bits=True"
                           % (stat_id,))
        mse, measured = self.bit_tables.table(stat_id)
        if measured != rule:
            raise ValueError("-bap mse: the tables of %r were measured under -c %s, this run clips with -c %s; collect "
                             "them under -c %s with collect_bits=True" % (stat_id, measured, rule, rule))
        m, stat = None, "max"
        if rule == "mse":
            m, prior = self.bit_tables.multipliers_of(stat_id)
            stat = "b" if prior == "laplace" else "std"
        scale = np.asarray(self._stat(stat_id, stat, "mean"), dtype=np.float32).reshape(-1)
        if mse.shape[0] != scale.size:
            raise ValueError("-bap mse: the table of %r has %d groups, the statistics %d channels"
                             % (stat_id, mse.shape[0], scale.size))
        return mse, scale, m

    def _use_params(self, tensor, stat_id, route):
        """The call site's `-sm use` parameters (``_UseParams``), solved once and kept on the device.  ``route``: the
        dispatch target's rule - "kld", "minmax" (per tensor), "minmax_pc" (per channel) or a clipping rule (per channel
        where the statistics are).  The key holds everything the solve reads."""
        positive = self._positive()
        key = ("use", stat_id, route, self.kld, self.clipping, self.num_bits, positive, self._pc_act(tensor),
               self.stats_kind, self.bit_alloc_act, self.bit_alloc_prior, self.bit_alloc_round, self.bit_alloc_target_act,
               str(tensor.device))
        hit = self._stat_cache.get(key)
        if hit is not None:
            return hit
        dev = tensor.device
        if route == "kld":   # int_quantizer.py:478-486 with :605-614, float64
            mn, mx, th, mean = (self._stat(stat_id, k, "mean") for k in ("min", "max", "kld_th", "mean"))
            rng, off = self.alpha2DeltaOffset(th, mx, mn, mean)
            preserve_zero = bool(self.enforce_true_zero and (off + rng) > 0 and off < 0)
            p = _UseParams(False, None if rng <= 0 else float(rng), float(off), None, preserve_zero)
        elif route == "minmax":   # int_quantizer.py:362-369: collected min/max ('mean' kind, or min-of-min / max-of-max)
            kmin, kmax = ("mean", "mean") if self.stats_kind == "mean" else ("min", "max")
            min_ = float(self._stat(stat_id, "min", kmin))
            max_ = float(self._stat(stat_id, "max", kmax))
            if positive:
                min_ = 0.0
            delta = np.float32(max_) - np.float32(min_)
            preserve_zero = bool((np.float32(min_) + delta) > 0 and min_ < 0)
            p = _UseParams(False, float(delta) if delta > 0 else None, min_, None, preserve_zero)
        elif route == "minmax_pc":   # int_quantizer.py:409-451
            c = tensor.shape[1]
            mn = torch.zeros(c, device=dev) if positive else _to_dev(
                np.asarray(self._stat(stat_id, "min", self.stats_kind), dtype=np.float32), dev).reshape(-1)
            mx = _to_dev(np.asarray(self._stat(stat_id, "max", self.stats_kind), dtype=np.float32), dev).reshape(-1)
            p = _UseParams(True, (mx - mn).contiguous(), mn.contiguous(), self._use_bits(stat_id, True, dev), None)
        else:   # int_quantizer.py:327-359 with :227-300
            mn, mx, mean = (self._stat(stat_id, k, "mean") for k in ("min", "max", "mean"))
            per_channel = self._pc_act(tensor) and np.size(mn) > 1 and np.size(mx) > 1
            alpha, bits = self._alpha_from_stats(stat_id, route, per_channel, dev)
            if per_channel:
                rng, off = self.alpha2DeltaOffset(alpha if isinstance(alpha, torch.Tensor) else np.asarray(alpha, dtype=np.float32),
                                                  np.asarray(mx, dtype=np.float32), np.asarray(mn, dtype=np.float32),
                                                  np.asarray(mean, dtype=np.float32))
                off_t = _to_dev(off, dev)
                max_t = off_t + _to_dev(rng, dev)            # :351
                off_t = off_t.reshape(-1).expand(tensor.shape[1]) if off_t.numel() == 1 else off_t.reshape(-1)
                p = _UseParams(True, (max_t.reshape(-1) - off_t).contiguous(), off_t.contiguous(), bits, None)
            else:
                rng, off = self.alpha2DeltaOffset(float(alpha), float(mx), float(mn), float(mean))
                p = _UseParams(False, torch.tensor(rng, dtype=torch.float32, device=dev),
                               torch.tensor(off, dtype=torch.float32, device=dev), None, None)
        self._stat_cache[key] = p
        return p

    def _clipping_params_from_stats(self, tensor, stat_id, clip_type):
        """(delta, offset, bits, per_channel) of the clipping rule ``clip_type`` at a call site: ``_use_params``' record."""
        p = self._use_params(tensor, stat_id, clip_type)
        return p.delta, p.offset, p.bits, p.per_channel

    def _alpha_from_stats(self, stat_id, clip_type, per_channel, dev):
        """(alpha, float32 [C] widths or None) of clipping ``clip_type`` from collected statistics (int_quantizer.py:227-325):
        fp32 per channel; per tensor in the reference's types (the Laplace alpha an fp32 device tensor, the others float64
        numpy / pandas values).  The widths are ``_use_bits``' (`-c mse` may take them from its joint tables)."""
        if clip_type == "mse":
            return self._mse_alpha_from_stats(stat_id, per_channel, dev)
        bits = self._use_bits(stat_id, per_channel, dev)
        return self._rule_alpha(stat_id, clip_type, per_channel, dev, bits), bits

    def _rule_alpha(self, stat_id, rule, per_channel, dev, bits):
        """alpha of ``_alpha_from_stats`` at the widths ``bits`` (None: ``num_bits``)."""
        positive = self._positive()
        if rule == "laplace":
            table_l = self.alpha_laplace_positive if positive else self.alpha_laplace
            b = self._stat(stat_id, "b", "mean")
            if bits is not None:
                factor = torch.tensor(np.array([table_l[int(v)] for v in bits.tolist()]), dtype=torch.float32, device=dev)
            else:
                factor = table_l[self.num_bits]
            return _to_dev(np.asarray(b, dtype=np.float32) if per_channel else b, dev) * factor
        if rule == "gaus":
            return self._stat(stat_id, "std", "mean") * (self.alpha_gaus_positive if positive else self.alpha_gaus)[self.num_bits]
        if rule == "lowp":   # `mix`'s no-clipping candidate
            return (self._stat(stat_id, "max", "mean") - self._stat(stat_id, "min", "mean")) / 2
        if rule == "mix":
            # int_quantizer.py:310-323, elementwise per tensor or per channel, with the reference's order: Gauss where
            # mse_gaus < mse_laplace, else Laplace; then lowp wherever mse_lowp < mse_gaus (even when Laplace beats both).
            # Ties keep the earlier choice; NaN errors (statistics collected without them) select Laplace.
            try:
                mse = {k: np.asarray(self._stat(stat_id, "mse_" + k, "mean"), dtype=np.float64) for k in ("lowp", "gaus", "laplace")}
            except KeyError:
                raise KeyError("-c mix needs the mse_* statistics of layer %r: collect them with collect_err=True" % (stat_id,))
            a = {k: self._rule_alpha(stat_id, k, per_channel, dev, bits) for k in ("laplace", "gaus", "lowp")}
            a = {k: v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v) for k, v in a.items()}
            alpha = np.where(mse["gaus"] < mse["laplace"], a["gaus"], a["laplace"])
            alpha = np.where(mse["lowp"] < mse["gaus"], a["lowp"], alpha)
            return alpha.astype(np.float32) if per_channel else alpha
        if "std" in rule:
            return float(rule.replace("std", "")) * self._stat(stat_id, "std", "mean")
        raise NotImplementedError("clipping %r is not supported with offline statistics" % rule)

    def _mse_alpha_from_stats(self, stat_id, per_channel, dev):
        """`-c mse`: (alpha, widths) with, per group, alpha = m* times the summary b (or std, for curves collected with
        mse_prior="gaus"), m* the multiplier at the minimum of the group's collected clipping-MSE curve (ties: the smaller
        multiplier) - fp32 per channel, float64 per tensor - and ``_use_bits``' widths; with `-baa -bap mse` a per-channel
        call site takes width and clipping value together from the joint tables (``_joint_alpha_from_stats``)."""
        if self.bit_alloc_prior == "mse" and self._allocates(per_channel):
            return self._joint_alpha_from_stats(stat_id, dev)
        if self.mse_curves is None:
            raise KeyError("-c mse needs the clipping-MSE curve of layer %r: collect it with collect_mse=True" % (stat_id,))
        m, prior = self.mse_curves.best(stat_id)
        scale = self._stat(stat_id, "b" if prior == "laplace" else "std", "mean")
        if per_channel:
            scale = np.asarray(scale, dtype=np.float32).reshape(-1)
            if m.size not in (1, scale.size):
                raise ValueError("-c mse: the curve of %r has %d groups, the statistics %d channels" % (stat_id, m.size, scale.size))
            return scale * m, self._use_bits(stat_id, per_channel, dev)
        if m.size != 1:
            raise ValueError("-c mse: the curve of %r is per channel (%d groups) but the layer is quantized per tensor"
                             % (stat_id, m.size))
        return float(scale) * float(m[0]), None

    def _joint_alpha_from_stats(self, stat_id, dev):
        """`-c mse -baa -bap mse`: (float32 [C] alpha, float32 [C] widths) of a per-channel, bit-allocated call site.  The
        widths are bit_alloc.allocate's on the layer's joint tables (bit_mse.pkl collected with collect_bits under -c
        mse: per channel and width, the error at the best multiplier), and alpha_c = m_w[c, w_c] * scale_c in fp32, scale
        the summary b (or std, for tables collected with mse_prior="gaus"), as `-c mse` forms it."""
        from .bit_alloc import allocate
        mse, scale, m = self._bit_table(stat_id, "mse")
        widths = allocate(mse, self.bit_alloc_target_act)
        return scale * m[np.arange(scale.size), widths], torch.tensor(widths, dtype=torch.float32, device=dev)

    def _use_apply(self, p, tensor, bias, table=None):
        """The one launch of use-mode parameters ``p``: per channel ``_quantize1`` (``table``: their parameter table, if
        the caller has it); per tensor the bias first (in place when the caller gave the tensor up), the `-bca` fallback,
        the empty-range pass-through of the compiled leaf, then ops.quantize1 (torch leaf) or ops.float2gemmlowp
        (compiled leaf)."""
        if p.per_channel:
            return self._quantize1(tensor, p.delta, p.offset, bits=p.bits, layout=self._nchw_layout(tensor), bias=bias,
                                   table=table)
        bca = self._bca is not None and tensor.dim() == 4
        if p.preserve_zero is None and bca:
            return self._quantize1(tensor, p.delta, p.offset, bias=bias)   # one parameter set, per-channel correction
        if bias is not None:
            tensor = tensor.add_(bias.view(1, -1, 1, 1)) if self.inplace else tensor + bias.view(1, -1, 1, 1)
        if p.preserve_zero is None:
            return ops.quantize1(tensor, p.delta, p.offset, self.num_bits, out=self._out(tensor))
        if p.delta is None:   # the leaf hands its input back (gemmlowp.cu:31-32)
            return torch.relu_(tensor) if (self._relu_follows and self.inplace) else (torch.relu(tensor) if self._relu_follows else tensor)
        res = ops.float2gemmlowp(tensor, p.delta, p.offset, self.num_bits, self.int_exp, p.preserve_zero, None,
                                 out=None if bca else self._out(tensor))
        return self.bias_correction_torch(tensor, res, bool(self._bca)) if bca else res

    # ------------------------------------------------------------------------------------------
    # dispatch targets
    # ------------------------------------------------------------------------------------------
    def gemmlowpClippingQuantize(self, tensor, id, tag="", stat_id=None, clip_type="laplace", bias=None):
        """ACIQ clipping, int_quantizer.py:327-359: per channel (pcq_a, 4-D, HW>1, C>1; fp32 parameter math,
        optional bit allocation) or per tensor (float64 parameter math)."""
        self._unsupported(stat_id)
        if stat_id is not None:
            return self._use_apply(self._use_params(tensor, stat_id, clip_type), tensor, bias)
        if self._fly_bits_site(tensor):
            return self._fly_bits(tensor, bias, clip_type)
        if clip_type == "mse":
            return self._fly_mse(tensor, bias)
        mode, k = self._range_mode(clip_type)
        if self._pc_act(tensor) and tensor.shape[1] > 1:
            hist = self._hist(tensor)  # the reference measures entropy in gemmlowpQuantizeActivationPerChannel (:442-445)
            res = self._launch(tensor, self._nchw_layout(tensor), channels_last=ops.cl_eligible(tensor),
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

    def _fly_mse(self, tensor, bias, max_ctas=0):
        """`-c mse` on the fly: each group (channel, as the on-the-fly ACIQ launch quantizes per channel, else the whole
        tensor) is clipped at the minimum of its own clipping-MSE curve over ``mse_candidates``.  A statistics-only launch
        configured like the ACIQ launch (scope, ``positive``, `-baa` widths), one ops.clip_mse_select launch pair that
        measures every candidate at the group's width and picks on the device, then the use-mode apply of the chosen
        parameters (``_use_apply``: block epilogue, deferred shortcut, pooling, slice write and `-bca` as in `-sm use`).
        ``bias`` is None: ``_bias_fusable`` has it added first.  Nothing goes through ``_stat_cache`` or back to the host."""
        if self.measure_entropy:
            raise NotImplementedError("-c mse on the fly does not measure entropy (-me): use -sm use with collected curves")
        cand = self.mse_candidates or _default_mse_candidates()
        positive = self._positive()
        if self._pc_act(tensor) and tensor.shape[1] > 1:
            layout = self._nchw_layout(tensor)
            cl = ops.cl_eligible(tensor)
            x = tensor if cl else tensor.contiguous()
            alloc = self._allocates(True)
            table = ops.fused(x, layout, stats_only=True, channels_last=cl, num_bits=self.num_bits, positive=positive,
                              bit_alloc=self.bit_alloc_act, bit_alloc_prior=self._prior(),
                              bit_alloc_round=self.bit_alloc_round, bit_alloc_target=self.bit_alloc_target_act)
            _, choice, given, chosen = ops.clip_mse_select(x, table, layout, cl, self.num_bits, positive,
                                                           cand.mult(tensor.device), prior=cand.prior, bit_alloc=alloc,
                                                           solve_f64=False, max_ctas=max_ctas)
            p = _UseParams(True, given[0], given[1], given[2] if alloc else None, None)
        else:
            x = tensor if ops.dense(tensor) else tensor.contiguous()
            layout = (1, 1, x.numel())
            table = ops.fused(x, layout, stats_only=True, num_bits=self.num_bits, positive=positive, any_dense_format=True)
            _, choice, given, chosen = ops.clip_mse_select(x, table, layout, False, self.num_bits, positive,
                                                           cand.mult(tensor.device), prior=cand.prior, solve_f64=True,
                                                           max_ctas=max_ctas)
            p = _UseParams(False, given[0, 0], given[1, 0], None, None)
        if self.export_stats:
            self.last_stats, self.last_clip_choice = chosen, choice
        return self._use_apply(p, tensor, bias, table=chosen)

    def _fly_bits(self, tensor, bias, rule, max_ctas=0):
        """`-baa -bap mse` on the fly (``fly_bits``): the channels of a per-channel, bit-allocated activation get the
        widths that minimise the sum of their own measured errors for ``bit_alloc_target_act`` bits per channel, the
        allocation `-sm use` makes from tables collected with collect_bits under clipping ``rule``.  A statistics-only
        launch without allocation (every candidate brings its own width), the candidates of each width 0..8 - those of
        statistics.bit_candidates through ops.clip_mse, or under -c mse every width times ``mse_candidates`` through
        ops.clip_mse_grid - then one ops.allocate_select, and the use-mode apply of its parameters (``_use_apply``: block
        epilogue, deferred shortcut, pooling, slice write and `-bca` as in `-sm use`).  ``bias`` is None: ``_bias_fusable``
        has it added first.  Nothing goes through ``_stat_cache`` or back to the host."""
        if self.measure_entropy:
            raise NotImplementedError("-baa -bap mse on the fly (fly_bits) does not measure entropy (-me)")
        positive = self._positive()
        layout = self._nchw_layout(tensor)
        cl = ops.cl_eligible(tensor)
        x = tensor if cl else tensor.contiguous()
        dev = tensor.device
        table = ops.fused(x, layout, stats_only=True, channels_last=cl, num_bits=8)
        if rule == "mse":
            cand = self.mse_candidates or _default_mse_candidates()
            mult = cand.mult(dev)
            sums, params = ops.clip_mse_grid(x, table, layout, cl, self.num_bits, positive, mult, range(9),
                                             prior=cand.prior, solve_f64=False, want_params=True, max_ctas=max_ctas)
        else:
            cand = _bit_candidates(rule, positive, self.num_bits)
            mult = None
            sums, params = ops.clip_mse(x, table, layout, cl, self.num_bits, positive, cand.mult(dev), prior=cand.prior,
                                        widths=range(9), solve_f64=False, want_params=True, max_ctas=max_ctas)
        _, choice, given, chosen = ops.allocate_select(sums, params, table, self.bit_alloc_target_act, multipliers=mult)
        if self.export_stats:
            self.last_stats, self.last_clip_choice = chosen, choice   # choice: None without a multiplier grid
        return self._use_apply(_UseParams(True, given[0], given[1], given[2], None), tensor, bias, table=chosen)

    def gemmlowpMinMaxQuantize(self, tensor, tag="", stat_id=None, weight_correction=None, bias=None):
        """Per-tensor min/max range through the compiled-leaf arithmetic, int_quantizer.py:361-379 + :605-614.
        Activations (tag contains 'activation', not 'classifier') use the batch average of per-sample min/max."""
        self._unsupported(stat_id)
        if stat_id is not None:
            return self._use_apply(self._use_params(tensor, stat_id, "minmax"), tensor, bias)
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

    def gemmlowpKldQuantize(self, tensor, tag="", stat_id=None):
        """Collected KLD threshold as the clipping value, int_quantizer.py:478-486: ('mean' kind) min / max / kld_th / mean
        -> alpha2DeltaOffset -> the compiled leaf, one apply-only launch.  The float64 arithmetic and the preserve-zero
        test of __gemmlowpQuantize__ run once per (layer, configuration); the leaf gets them as fp32 scalars, like the
        reference's pybind call."""
        if stat_id is None or self.sm is None:
            raise RuntimeError("KLD quantization (-kld) needs collected statistics: call with stat_id and a statistics "
                               "manager attached (q.sm, `-sm use`)")
        return self._use_apply(self._use_params(tensor, stat_id, "kld"), tensor, None)

    def gemmlowpQuantizeActivationPerChannel(self, tensor, id, tag="", stat_id=None, min_=None, max_=None, bias=None):
        """Per-channel min/max (0 lower bound when positive) with optional bit allocation, int_quantizer.py:409-451."""
        self._unsupported(stat_id)
        layout = self._nchw_layout(tensor)
        if stat_id is not None and min_ is None and max_ is None:
            return self._use_apply(self._use_params(tensor, stat_id, "minmax_pc"), tensor, bias)
        if min_ is None and max_ is None and self._fly_bits_site(tensor):
            return self._fly_bits(tensor, bias, "no")
        if min_ is None and max_ is None:
            hist = self._hist(tensor)
            res = self._launch(tensor, layout, channels_last=ops.cl_eligible(tensor),
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
            refuse_clip_weight(self.clip_weight, bounds=True)
            t = tensor.reshape(rows, -1)
            mn = _to_dev(min_, tensor.device) if min_ is not None else t.min(-1)[0]
            mx = _to_dev(max_, tensor.device) if max_ is not None else t.max(-1)[0]
            bits = None
            if self.bit_alloc_weight and self.num_bits <= 4:
                if self.bit_alloc_prior == "mse":
                    raise NotImplementedError("-baw -bap mse measures the weight's own min/max range: explicit min_ / max_ "
                                              "bounds are not supported")
                bits = self.get_bits_alloc_fixed_target(t.std(-1), self.bit_alloc_target_weight, self.bit_alloc_round)
            return ops.quantize1(tensor, mx - mn, mn, self.num_bits, bits=bits, layout=layout)
        bc, vc = weight_correction if weight_correction is not None else (False, False)
        if self.clip_weight == "mse":
            return self._clip_mse_weights(tensor, id, layout, bc, vc)
        if self.bit_alloc_weight and self.num_bits <= 4 and self.bit_alloc_prior == "mse":
            return self._mse_weights(tensor, id, layout, bc, vc)
        hist = self._hist(tensor)
        res = self._fused(tensor, layout, scope=L.SCOPE_GROUP, range_mode=L.RANGE_MINMAX, leaf=L.LEAF_TORCH,
                        num_bits=self.num_bits, positive=False, bit_alloc=self.bit_alloc_weight,
                        bit_alloc_prior=L.PRIOR_STD, bit_alloc_round=self.bit_alloc_round,
                        bit_alloc_target=self.bit_alloc_target_weight, bias_corr=bc, var_corr=vc, hist=hist)
        self._log_entropy(hist, id, "avg.entropy.weight", tensor.numel())
        return res

    def _mse_weights(self, tensor, id, layout, bias_corr, var_corr):
        """`-baw -bap mse`: per output channel the min/max range, at the widths that minimise the weight's measured
        squared error for the budget of bit_alloc_target_weight bits per channel: a statistics-only launch, one
        ops.clip_mse over widths 0..8, bit_alloc.allocate on the host, then one given-parameter launch (with `-me`, its
        grid gives the entropy).  The bias and variance corrections follow as stock torch ops on the NCHW-ordered weight
        (a channels-last weight is read in that order by every launch here, and the result comes back in it)."""
        from .bit_alloc import MAX_BITS, allocate
        table = ops.fused(tensor, layout, num_bits=8, stats_only=True)
        widths = list(range(MAX_BITS + 1))
        sse = ops.clip_mse(tensor, table, layout, False, self.num_bits, False, [0.0] * len(widths), prior="minmax",
                           widths=widths, solve_f64=False)
        bits = torch.tensor(allocate(sse[:, 1:], self.bit_alloc_target_weight), dtype=torch.float32, device=tensor.device)
        mn, mx = table[:, 0].contiguous(), table[:, 1]
        if self.measure_entropy:
            res, grid = ops.quantize1(tensor, (mx - mn).contiguous(), mn, self.num_bits, bits=bits, layout=layout,
                                      want_grid=True)
            hist = torch.bincount(grid.flatten().to(torch.int64).clamp_(0, 255), minlength=256)
            self._log_entropy(hist, id, "avg.entropy.weight", tensor.numel())
        else:
            res = ops.quantize1(tensor, (mx - mn).contiguous(), mn, self.num_bits, bits=bits, layout=layout)
        if bias_corr or var_corr:
            from .manager import QuantizationManagerInference
            res = QuantizationManagerInference._weight_correction_torch(tensor.contiguous(), res.contiguous(), bias_corr,
                                                                        var_corr)
        return res

    def _clip_mse_weights(self, tensor, id, layout, bias_corr, var_corr, max_ctas=0):
        """`clip_weight="mse"`: per output channel the candidate with the least measured squared error among the min/max
        range (first: it wins exact ties) and the clipping values of ``weight_mse`` (in their order; NaN never wins), at
        the channel's width - ``num_bits``; with `-baw`, the width the default launch's bit allocation gives it, or under
        `-bap mse` the widths fqb200_allocate_widths picks from the per-width best errors.  A statistics-only launch, the
        candidates' errors and parameters (ops.clip_mse_grid, ops.clip_mse with prior "minmax"), the selection as device
        tensor ops, and one ops.quantize_weights_given launch with the call's corrections and `-me` histogram, which runs
        the chosen parameters exactly as they were measured.  A channels-last weight is read in NCHW order throughout and
        the result comes back in it.  Nothing is read back to the host."""
        wm = self.weight_mse
        dev = tensor.device
        g = layout[1]
        alloc = bool(self.bit_alloc_weight and self.num_bits <= 4)
        table = ops.fused(tensor, layout, num_bits=self.num_bits, bit_alloc=self.bit_alloc_weight,
                          bit_alloc_prior=L.PRIOR_STD, bit_alloc_round=self.bit_alloc_round,
                          bit_alloc_target=self.bit_alloc_target_weight, stats_only=True)
        widths = list(range(9)) if alloc else [self.num_bits]
        nw = len(widths)
        mult = wm.mult(dev)
        m = mult.numel()
        grid, gp = ops.clip_mse_grid(tensor, table, layout, False, self.num_bits, False, mult, widths, prior=wm.prior,
                                     want_params=True, max_ctas=max_ctas)
        mm, mp = ops.clip_mse(tensor, table, layout, False, self.num_bits, False, torch.zeros(nw, device=dev),
                              prior="minmax", widths=widths, want_params=True, max_ctas=max_ctas)
        err = torch.cat([mm[:, 1:].reshape(g, nw, 1), grid[:, 1:].reshape(g, nw, m)], 2)
        par = torch.cat([mp.reshape(g, nw, 1, 6), gp.reshape(g, nw, m, 6)], 2)
        pick, best = best_candidates(err)
        if not alloc:
            wi = torch.zeros(g, dtype=torch.int64, device=dev)
        elif self.bit_alloc_prior == "mse":
            wi = ops.allocate_widths(best, self.bit_alloc_target_weight, wm.status(dev)).long()
        else:
            wi = table[:, 7].long()
        k = pick.gather(1, wi.unsqueeze(1)).squeeze(1)
        p = par[torch.arange(g, device=dev), wi, k]
        bits = p[:, 2].contiguous() if alloc else None
        hist = self._hist(tensor)
        res = ops.quantize_weights_given(tensor, p[:, 0].contiguous(), p[:, 1].contiguous(), self.num_bits, bits=bits,
                                         bias_corr=bias_corr, var_corr=var_corr, hist=hist)
        self._log_entropy(hist, id, "avg.entropy.weight", tensor.numel())
        if self.export_stats:   # per channel: the chosen candidate's error, min/max's error at its width, the width
            self.last_weight_mse = (best.gather(1, wi.unsqueeze(1)).squeeze(1), mm[:, 1:].gather(1, wi.unsqueeze(1)).squeeze(1),
                                    p[:, 2])
        if wm.report is not None:
            nan = torch.full((), math.nan, dtype=torch.float64, device=dev)
            ref_bits, ref_sse = nan, nan
            if alloc and self.bit_alloc_prior == "mse":   # today's min/max-only allocation for the same budget
                wmm = ops.allocate_widths(mm[:, 1:], self.bit_alloc_target_weight, wm.status(dev)).long()
                ref_bits, ref_sse = wmm.sum().double(), mm[:, 1:].gather(1, wmm.unsqueeze(1)).sum()
            wm.add(id, g, tensor.numel(), torch.stack([
                p[:, 2].double().sum(), mm[:, 1:].gather(1, wi.unsqueeze(1)).sum(), best.gather(1, wi.unsqueeze(1)).sum(),
                (k == 0).sum().double(), ref_bits, ref_sse]))
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

    def _mid_tread_bins(self):
        if self.bit_alloc_prior == "mse":
            refuse_bap_mse(mid_tread=True)

    def mid_tread_quantize_weights_per_channel(self, tensor, id, weight_correction=None):
        self._mid_tread_bins()
        rows = tensor.shape[0]
        bc, vc = weight_correction if weight_correction is not None else (False, False)
        if self.measure_entropy:
            self._log_mt_entropy(self._mid_tread_entropy_torch(tensor.reshape(rows, -1), self.bit_alloc_target_weight, False, True),
                                 id, "avg.entropy.weight", tensor.numel())
        return self._fused(tensor, (1, rows, tensor.numel() // rows), leaf=L.LEAF_MIDTREAD, positive=False,
                         mt_target=self.bit_alloc_target_weight, mt_clip=False, bias_corr=bc, var_corr=vc)

    def mid_tread_quantize_activation(self, tensor, id, bias=None):
        self._mid_tread_bins()
        if self._pc_act(tensor):
            return self.mid_tread_quantize_activation_per_channel(tensor, id, bias=bias)
        if bias is not None:
            tensor = tensor + bias.view((1, -1) + (1,) * (tensor.dim() - 2))
        return self._fused(tensor, (1, 1, tensor.numel()), leaf=L.LEAF_MIDTREAD, positive=self._positive(),
                         mt_target=self.bit_alloc_target_act, mt_clip=True, out=self._out(tensor))

    def mid_tread_quantize_activation_per_channel(self, tensor, id, bias=None):
        self._mid_tread_bins()
        layout = self._nchw_layout(tensor)
        kw = dict(leaf=L.LEAF_MIDTREAD, positive=self._positive(), mt_target=self.bit_alloc_target_act, mt_clip=True, bias=bias,
                  out=self._out(tensor), channels_last=ops.cl_eligible(tensor))
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
        self._mid_tread_bins()
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
        if self._allocates(per_channel) and self.bit_alloc_prior == "mse":
            refuse_bap_mse(needs_use=True)
        stats = self.__act_stats_perchannel__ if per_channel else self.__act_stats__
        b = stats(tensor, ["b"])["b"]
        table = self.alpha_laplace_positive if self._positive() else self.alpha_laplace
        if self._allocates(per_channel):
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
        """int_quantizer.py:302-325.  ``mix`` needs collected statistics (``stat_id`` and ``sm``), as in the reference;
        so does ``mse``, this package's extension."""
        if clip_type == "mix":
            if stat_id is None or self.sm is None:
                raise NotImplementedError("clipping 'mix' chooses by collected errors: it needs stat_id and a statistics "
                                          "manager (-sm use with statistics collected with collect_err=True)")
            return self._alpha_from_stats(stat_id, "mix", per_channel, tensor.device)[0]
        if clip_type == "mse":
            if stat_id is None or self.sm is None:
                raise NotImplementedError("clipping 'mse' clips at the minimum of collected curves: it needs stat_id and a "
                                          "statistics manager (-sm use with curves collected with collect_mse=True)")
            return self._mse_alpha_from_stats(stat_id, per_channel, tensor.device)[0]
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
