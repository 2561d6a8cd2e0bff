"""Offline calibration statistics (`-sm collect` / `-sm use`): mirrors of the reference's
``StatisticManager`` (per tensor, CSV; statistic_manager.py:15-178) and ``StatisticManagerPerChannel`` (per channel,
pickle; statistic_manager_perchannel.py:17-174) with the same on-disk formats, so statistics collected by either
implementation can be used by the other:

    <base>/statistics/<folder>/<id>.csv                         one row per batch, columns = statistic names
    <base>/statistics/<folder>/<folder>_summary.csv            index = id, columns internal_name, {min,mean,max}_<stat>, dim
    <base>/statistics/per_channel/<folder>/<folder>_statistics_perchannel_summary.pkl
                                                               {id: DataFrame[{min,mean,max}_<stat>], one row per channel}

``base`` defaults to ``~/mxt-sim`` like the reference (override with the constructor argument or $FQB200_STATS_DIR).

Collect mode is an offline, one-time pass.  The five statistics the quantizers consume in use mode (min, max, mean,
b, std) come from ONE statistics-only launch of the fused kernel per hooked tensor; the diagnostic columns the
reference also writes (kurtosis, mean_abs, std_pos) are computed with plain torch ops; the error columns
(mse_*/cos_*) are NaN exactly as in the reference's own collect runs (it never passes quantized tensors there), unless
the caller hands ``save_tensor_stats`` a ``ClipErrConfig``: then one ops.clip_error launch per hooked tensor fills them
with the errors of the three candidates `-c mix` chooses between (lowp, gaus, laplace), each configured like the
tensor's use-mode quantizer.
With ``kld_threshold`` the per-tensor manager adds the ``kld_th`` column: the max over the samples of the KL-divergence
threshold (ops.kld_threshold, three launches and one read-back per hooked tensor).

``MeasureStatistics`` is the activation norm measurement (`-ms`, distance_stats.py:15-54):

    <base>/distance/<folder>/distance.csv                       columns = ids in first-call order, one row per sample

Each hooked tensor costs one ops.sample_sumsq launch; the results stay on the device until ``__exit__``.

``AngleStatistics`` is its sibling for the pairwise angles between samples (angle_stats.py:22-80):

    <base>/angle/<folder>/angle.pkl      {id: DataFrame [calls * N, N] (the per-call matrices stacked), ..., 'target': labels}

Each hooked tensor costs one ops.sample_angles launch pair; the float32 [N, N] matrices stay on the device until
``__exit__`` (1 MB per measured tensor and batch at N = 512: about 54 MB per ResNet-50 batch).

``NoiseStatistics`` is the quantization-noise measurement (measure_statistics.py:19-99): the error each call site's
quantizer put into its output, with the moments of the layer's input, output and weight:

    <base>/noise/<folder>/<id>.csv       columns NOISE_COLUMNS, one row per sample in call order

Each hooked tensor costs two ops.sample_noise launch pairs (output with its quantized form, input) and each weight one,
once; the float64 sums stay on the device until ``__exit__`` (72 B per sample and call).

``ClipMseStatistics`` is the clipping-MSE curve of every collect call site (`collect_mse`; the simulation of the
reference's mse_analysis.py on real activations, with the quantizer the call site uses in `-sm use`), and what `-c mse`
reads back in use mode:

    <base>/clip_mse/<folder>/clip_mse.pkl   {"multipliers", "prior", id: DataFrame[count, b, std, bits, mse_<k>...], one
                                            row per group (channel of a per-channel quantizer, else the whole tensor)}
    <base>/clip_mse/<folder>/curve.csv      id, internal_name, multiplier, mse, mse_laplace_analytic, mse_gaus_analytic

Each hooked tensor costs one statistics-only launch and one ops.clip_mse launch pair; the sums stay on the device until
``__exit__``, which reads everything back in one copy.

``BitMseStatistics`` is the per-channel error table of every collect call site that `-sm use` quantizes per channel with
bit allocation (`collect_bits`): the error the call site's quantizer makes on each channel at every width 0..8, and what
`-bap mse` allocates from in use mode:

    <base>/bit_mse/<folder>/bit_mse.pkl     {"rule", id: DataFrame[count, b, std, positive, mse_w0 .. mse_w8], one row
                                            per channel}
    <base>/bit_mse/<folder>/alloc.csv       id, internal_name, groups, target, and bits_* / mse_* (bit sum, per-element
                                            MSE) of the uniform width, the analytic allocation and the measured one

It costs the same as ``ClipMseStatistics`` with 9 candidates.
"""
import collections
import functools
import os
import pickle
import re
import shutil

import numpy as np
import torch

from . import ops

__all__ = ["StatisticManager", "StatisticManagerPerChannel", "MeasureStatistics", "AngleStatistics", "NoiseStatistics",
           "ClipErrConfig", "ClipMseStatistics", "MSE_MULTIPLIERS", "MseCandidates", "BitMseStatistics", "bit_candidates",
           "default_base_dir"]


def default_base_dir():
    return os.environ.get("FQB200_STATS_DIR") or os.path.join(os.path.expanduser("~"), "mxt-sim")


def _fresh_folder(folder):
    """Create ``folder`` empty: a collect run replaces the files of an earlier one."""
    if os.path.exists(folder):
        shutil.rmtree(folder)
    os.makedirs(folder)


def sorted_nicely(keys):
    """Natural sort (conv2 before conv10), utils/misc.py:77-88."""
    conv = lambda t: int(t) if t.isdigit() else t
    return sorted(keys, key=lambda k: [conv(c) for c in re.split("([0-9]+)", k)])


_ERR_COLUMNS = ["mse_lowp", "mse_gaus", "mse_laplace", "cos_lowp", "cos_gaus", "cos_laplace"]

# The quantizer of one call site, as far as the measurements need it (IntQuantizer.clip_err_config): its bit width, its
# positive range (half_range / force_positive), whether it quantizes this tensor per channel and its bit allocation (per
# channel with num_bits <= 4 only; prior PRIOR_STD / PRIOR_B).
ClipErrConfig = collections.namedtuple("ClipErrConfig", "num_bits positive per_channel bit_alloc bit_alloc_prior "
                                                        "bit_alloc_round bit_alloc_target")


def _stats_table(t, cfg, channels_last):
    """(``t`` in the memory order the launches read, layout, channels-last flag, table) of the statistics-only launch of
    the quantizer ``cfg`` describes: per channel (with ``cfg``'s bit allocation) in place on a channels-last ``t`` when
    ``channels_last`` allows it, else on the NCHW tensor; per tensor in any dense memory order.  The candidate launches
    read the statistics (columns 0..4) and, with bit allocation, the widths (column 7) of the table; without allocation
    the table is solved at 8 bits."""
    if not cfg.per_channel:
        if not ops.dense(t):
            t = t.contiguous()
        layout = (1, 1, t.numel())
        return t, layout, False, ops.fused(t, layout, positive=cfg.positive, stats_only=True, any_dense_format=True)
    n, c = t.shape[0], t.shape[1]
    layout = (n, c, t.numel() // (n * c))
    cl = channels_last and ops.cl_eligible(t, layout)
    if not cl:
        t = t.contiguous()
    return t, layout, cl, ops.fused(t, layout, num_bits=cfg.num_bits if cfg.bit_alloc else 8, positive=cfg.positive,
                                    bit_alloc=cfg.bit_alloc, bit_alloc_prior=cfg.bit_alloc_prior,
                                    bit_alloc_round=cfg.bit_alloc_round, bit_alloc_target=cfg.bit_alloc_target,
                                    stats_only=True, channels_last=cl)


def _curve(t, cfg, cand, select=False, max_ctas=0):
    """The clipping-MSE curve of the quantizer ``cfg`` describes on ``t`` over the candidates ``cand`` (an
    MseCandidates), each at the group's width: ``_stats_table``'s (tensor, layout, channels-last flag, table) and the
    result of the candidate launch - ops.clip_mse's sums, or with ``select`` ops.clip_mse_select's (sums, choice, given
    parameters, parameter table).  What `collect_mse` accumulates and `-c mse` on the fly chooses from."""
    t, layout, cl, table = _stats_table(t, cfg, True)
    launch = ops.clip_mse_select if select else ops.clip_mse
    return t, layout, cl, table, launch(t, table, layout, cl, cfg.num_bits, cfg.positive, cand.mult(t.device),
                                        prior=cand.prior, bit_alloc=cfg.bit_alloc, solve_f64=not cfg.per_channel,
                                        max_ctas=max_ctas)


def _width_tables(t, cfg, rule, cand, want_params=False, max_ctas=0):
    """The per-channel error tables of the quantizer ``cfg`` describes on ``t`` at every width 0..8 under the clipping
    ``rule``: ``_stats_table``'s (tensor, layout, channels-last flag, table) of an 8-bit table without allocation (every
    candidate brings its own width) and the result of the candidate launch - ops.clip_mse over the candidates of
    ``bit_candidates``, or under rule "mse" ops.clip_mse_grid over widths 0..8 times ``cand`` (an MseCandidates; unused
    under the other rules); with ``want_params`` (sums, parameters).  What `collect_bits` accumulates and `fly_bits`
    allocates from."""
    t, layout, cl, table = _stats_table(t, cfg._replace(bit_alloc=False), True)
    if rule == "mse":
        out = ops.clip_mse_grid(t, table, layout, cl, cfg.num_bits, cfg.positive, cand.mult(t.device), range(9),
                                prior=cand.prior, solve_f64=False, want_params=want_params, max_ctas=max_ctas)
    else:
        widths = _width_candidates(rule, cfg.positive, cfg.num_bits)
        out = ops.clip_mse(t, table, layout, cl, cfg.num_bits, cfg.positive, widths.mult(t.device), prior=widths.prior,
                           widths=range(9), solve_f64=False, want_params=want_params, max_ctas=max_ctas)
    return t, layout, cl, table, out


def _clip_sums(t, cfg, per_sample_channel):
    """float64 ops.clip_error sums (columns as there) of the contiguous ``t`` for the candidates ``cfg`` describes:
    [1, 10] over the whole tensor, or with ``per_sample_channel`` [N, C, 10] per (sample, channel) - the per-channel
    manager needs the per-sample norms of the reference's cos_sim(dims=[-1, 0]).  The candidates' statistics are those
    of the on-the-fly launch of that quantizer (``_stats_table``); a per-(sample, channel) launch gets that table
    repeated for every group, and a per-channel quantizer's errors over the whole tensor are the sum of its groups'."""
    t, layout, _, table = _stats_table(t, cfg, False)
    if not (per_sample_channel or cfg.per_channel):
        return ops.clip_error(t, table, layout, False, cfg.num_bits, cfg.positive, solve_f64=True)
    n, c = t.shape[0], t.shape[1]
    table = table.repeat(n, 1) if cfg.per_channel else table.expand(n * c, -1).contiguous()
    sums = ops.clip_error(t, table, (1, n * c, t.numel() // (n * c)), False, cfg.num_bits, cfg.positive,
                          bit_alloc=cfg.bit_alloc, solve_f64=not cfg.per_channel).view(n, c, 10)
    return sums if per_sample_channel else sums.sum((0, 1)).view(1, -1)


def _clip_errors(sums, count, per_channel):
    """{mse_k, cos_k} float32 device tensors from _clip_sums: per tensor ([1, 10]) mse = sum (x - q)^2 / count and
    cos = sum x q / (sqrt(sum x^2) sqrt(sum q^2)) (statistic_manager.py:83-103); per channel ([N, C, 10]) mse over the
    channel's N * HW elements and the reference's cos_sim(dims=[-1, 0]): sum_n sum_hw x q /
    (sqrt(sum_n sqrt(sum_hw x^2)) sqrt(sum_n sqrt(sum_hw q^2))) (statistic_manager_perchannel.py:80-100, utils/misc.py)."""
    res = {}
    for k, name in enumerate(ops.CLIP_ERROR_CANDIDATES):
        if per_channel:
            res["mse_" + name] = (sums[:, :, 1 + k].sum(0) / count).float()
            res["cos_" + name] = (sums[:, :, 4 + k].sum(0) / (sums[:, :, 0].sqrt().sum(0).sqrt()
                                                              * sums[:, :, 7 + k].sqrt().sum(0).sqrt())).float()
        else:
            res["mse_" + name] = (sums[:, 1 + k] / count).float()
            res["cos_" + name] = (sums[:, 4 + k] / (sums[:, 0].sqrt() * sums[:, 7 + k].sqrt())).float()
    return res


class StatisticManager(object):
    """Per-tensor statistics (statistic_manager.py:15-178)."""

    def __init__(self, folder, load_stats, stats=None, batch_avg=False, kld_threshold=False, collect_err=True, base_dir=None):
        self.name = folder
        self.folder = os.path.join(base_dir or default_base_dir(), "statistics", folder)
        self.stats_names = list(stats) if stats is not None else ["max", "min", "std", "mean", "kurtosis", "mean_abs", "b", "dim"]
        self.batch_avg = batch_avg
        if collect_err:
            self.stats_names += _ERR_COLUMNS
        self.kld_threshold = kld_threshold
        if kld_threshold:
            self.stats_names.append("kld_th")
        self.stats = {}
        self.metadata = {}
        self.save_stats = not load_stats
        self.stats_df = None
        if load_stats:
            import pandas as pd
            path = os.path.join(self.folder, "%s_summary.csv" % self.name)
            if not os.path.exists(path):
                raise FileNotFoundError("no collected statistics at %s (run with stats_mode='collect' first)" % path)
            self.stats_df = pd.read_csv(path, index_col=0)

    # -- collect ---------------------------------------------------------------------------------------
    def save_tensor_stats(self, tensor, tag, id, tensors_q=None, force_global_min_max=False, clip_err=None):
        """One row of statistics for this batch (statistic_manager.py:47-122).  ``clip_err`` (a ClipErrConfig): fill the
        mse_* / cos_* columns with the errors of the `-c mix` candidates configured like that (else they are NaN)."""
        t = tensor.detach().contiguous()
        n = t.shape[0]
        st = ops.fused(t, (1, 1, t.numel()), stats_only=True)[0]  # min max mean b std over the whole tensor
        glob = {"min": st[0], "max": st[1], "mean": st[2], "b": st[3], "std": st[4]}
        err = None
        if clip_err is not None and any(c in self.stats_names for c in _ERR_COLUMNS):
            e = _clip_errors(_clip_sums(t, clip_err, False), float(t.numel()), False)
            err = dict(zip(_ERR_COLUMNS, torch.cat([e[c] for c in _ERR_COLUMNS]).cpu().tolist()))   # one copy
        if self.batch_avg and not force_global_min_max:
            per = ops.fused(t, (1, n, t.numel() // n), stats_only=True)
            glob["min"], glob["max"] = per[:, 0].mean(), per[:, 1].mean()
        row = []
        flat = t.view(-1)
        for sn in self.stats_names:
            if sn in glob:
                v = glob[sn]
            elif sn == "kurtosis":
                v = torch.mean(((flat - glob["mean"]) / glob["std"]) ** 4) - 3
            elif sn == "mean_abs":
                v = torch.mean(flat.abs())
            elif sn == "dim":
                v = flat.numel()
            elif sn == "kld_th":
                v = ops.kld_threshold(t)[0].max()   # the max of the per-sample thresholds (NaN propagates, as np.max)
            elif err is not None:  # mse_* / cos_*
                v = err[sn]
            else:  # mse_* / cos_*: the reference writes NaN when no quantized tensors are handed in
                v = float("nan")
            row.append(float(v))
        arr = np.asarray(row, dtype=np.float64).reshape(1, -1)
        if id in self.stats:
            self.stats[id] = np.concatenate([self.stats[id], arr])
        else:
            self.stats[id] = arr
            self.metadata[id] = tag

    # -- use -------------------------------------------------------------------------------------------
    def get_tensor_stat(self, id, stat, kind="mean"):
        if self.stats_df is None:
            return None
        return self.stats_df.loc[id, "%s_%s" % (kind, stat)]

    def get_tensor_stats(self, id, kind=None):
        kind = kind or {"min": "mean", "max": "mean", "mean": "mean", "std": "mean", "mean_abs": "mean", "b": "mean"}
        if self.stats_df is None:
            return (None,) * 6
        return tuple(self.stats_df.loc[id, "%s_%s" % (kind[s], s)] for s in ("min", "max", "mean", "std", "mean_abs", "b"))

    # -- persistence (statistic_manager.py:146-178) ----------------------------------------------------------
    def __exit__(self, *args):
        if not self.save_stats:
            return
        import pandas as pd
        _fresh_folder(self.folder)
        frames = {}
        for s_id, data in self.stats.items():
            df = pd.DataFrame(columns=self.stats_names, data=data)
            df.to_csv(os.path.join(self.folder, "%s.csv" % s_id), index=False)
            frames[s_id] = df
        cols = []
        for c in self.stats_names:
            cols += ["min_%s" % c, "mean_%s" % c, "max_%s" % c]
        summary = pd.DataFrame(columns=["internal_name"] + cols)
        for s_id in sorted_nicely(frames.keys()):
            summary.loc[s_id, "internal_name"] = self.metadata[s_id]
            for c in self.stats_names:
                summary.loc[s_id, "min_%s" % c] = frames[s_id][c].min()
                summary.loc[s_id, "mean_%s" % c] = frames[s_id][c].mean()
                summary.loc[s_id, "max_%s" % c] = frames[s_id][c].max()
            summary.loc[s_id, "dim"] = frames[s_id]["dim"][0] if "dim" in frames[s_id] else np.nan
        summary.to_csv(os.path.join(self.folder, "%s_summary.csv" % self.name), index=True)

    def __enter__(self):
        return self


class StatisticManagerPerChannel(object):
    """Per-channel statistics of [N, C, H, W] activations (statistic_manager_perchannel.py:17-174)."""

    def __init__(self, folder, load_stats, stats=None, batch_avg=False, collect_err=False, base_dir=None):
        self.name = folder
        self.folder = os.path.join(base_dir or default_base_dir(), "statistics/per_channel", folder)
        self.stats_names = list(stats) if stats is not None else ["max", "min", "std", "mean", "kurtosis", "b", "std_pos"]
        self.batch_avg = batch_avg
        if collect_err:
            self.stats_names += _ERR_COLUMNS
        self.save_stats = not load_stats
        self.stats = {}
        if load_stats:
            path = os.path.join(self.folder, "%s_statistics_perchannel_summary.pkl" % self.name)
            if not os.path.exists(path):
                raise FileNotFoundError("no collected per-channel statistics at %s" % path)
            with open(path, "rb") as f:
                self.stats = pickle.load(f)

    def save_tensor_stats(self, tensor, tag, id, tensors_q=None, force_global_min_max=False, clip_err=None):
        """Per-channel rows for this batch (statistic_manager_perchannel.py:45-122); FC / 1x1 tensors are skipped.
        ``clip_err`` (a ClipErrConfig): fill the mse_* / cos_* rows, when the manager has those columns (collect_err), with
        the per-channel errors of the `-c mix` candidates configured like that."""
        if tensor.dim() < 3 or (tensor.shape[2] == 1 and tensor.shape[3] == 1):
            return
        t = tensor.detach().contiguous()
        n, c = t.shape[0], t.shape[1]
        hw = t.numel() // (n * c)
        st = ops.fused(t, (n, c, hw), stats_only=True)  # [C, 12]: min max mean b std ...
        vals = {"min": st[:, 0], "max": st[:, 1], "mean": st[:, 2], "b": st[:, 3], "std": st[:, 4]}
        if clip_err is not None and any(s in self.stats_names for s in _ERR_COLUMNS):
            vals.update(_clip_errors(_clip_sums(t, clip_err, True), float(n * hw), True))
        if not force_global_min_max:
            per = ops.fused(t, (1, n * c, hw), stats_only=True).view(n, c, -1)  # per (n, c)
            if self.batch_avg:
                vals["max"], vals["min"] = per[:, :, 1].mean(0), per[:, :, 0].mean(0)
            else:
                vals["min"] = per[:, :, 0].min(0)[0]  # the reference's non-averaged min is the min over n of per-(n,c) minima
        tc = None
        for sn in self.stats_names:
            if sn in vals:
                v = vals[sn]
            elif sn in ("kurtosis", "std_pos"):
                if tc is None:
                    tc = t.transpose(0, 1).reshape(c, -1)  # offline diagnostics only: a transposed copy is fine here
                if sn == "kurtosis":
                    v = torch.mean(((tc - vals["mean"].unsqueeze(-1)) / vals["std"].unsqueeze(-1)) ** 4, dim=-1) - 3
                else:
                    v = torch.std(torch.relu(tc), dim=-1, unbiased=True)
            else:
                continue  # mse_* / cos_* need quantized tensors: skipped like the reference does
            v = v.detach().cpu().numpy()
            if sn.startswith("cos_"):   # statistic_manager_perchannel.py:113-115
                v = np.nan_to_num(v)
                v[v == 0] = 1.
            entry = self.stats.setdefault(id, {})
            entry[sn] = v if sn not in entry else np.vstack([entry[sn], v])

    def get_tensor_stat(self, id, stat, kind="mean"):
        if self.stats is None:
            return None
        return self.stats[id]["%s_%s" % (kind, stat)]

    def __exit__(self, *args):
        if not self.save_stats:
            return
        import pandas as pd
        _fresh_folder(self.folder)
        cols = []
        for c in self.stats_names:
            cols += ["min_%s" % c, "mean_%s" % c, "max_%s" % c]
        summary = {}
        for layer, entry in self.stats.items():
            df = pd.DataFrame(columns=cols)
            for s in self.stats_names:
                if s in entry:
                    t = entry[s]
                    multi = len(t.shape) > 1
                    df["min_%s" % s] = t.min(axis=0) if multi else [t.min(axis=0)]
                    df["mean_%s" % s] = t.mean(axis=0) if multi else [t.mean(axis=0)]
                    df["max_%s" % s] = t.max(axis=0) if multi else [t.max(axis=0)]
            summary[layer] = df
        with open(os.path.join(self.folder, "%s_statistics_perchannel_summary.pkl" % self.name), "wb") as f:
            pickle.dump(summary, f)

    def __enter__(self):
        return self


class MeasureStatistics(object):
    """Per-sample squared L2 norm of every measured tensor (distance_stats.py:15-54): ``save_measure(t, id)`` records
    sum(t[i]**2) for every sample i; ``__exit__`` writes them, rounded to float32 (the reference sums in float32), as one
    column per id in first-call order and one row per sample in call order."""

    def __init__(self, folder, base_dir=None):
        self.folder = os.path.join(base_dir or default_base_dir(), "distance", folder)
        self.stats = {}   # id -> float64 [N] tensors, one per call
        self.stats_names = ["dist"]

    def save_measure(self, tensor, id):
        t = tensor.detach()
        if t.is_cuda:
            d = ops.sample_sumsq(t)   # enqueued now: later in-place writes to the tensor come after it in stream order
        else:
            d = t.reshape(t.shape[0], -1).double().pow(2).sum(-1)
        self.stats.setdefault(id, []).append(d)

    def __enter__(self):
        return self

    def __exit__(self, *args):
        if not self.stats:
            return
        import pandas as pd
        cols = list(self.stats)
        per_id = [torch.cat(v) for v in self.stats.values()]
        rows = per_id[0].numel()
        if any(c.numel() != rows for c in per_id):
            raise ValueError("-ms: the measured ids saw different numbers of samples: %s"
                             % {k: c.numel() for k, c in zip(cols, per_id)})
        dev = per_id[0].device
        # one device-to-host copy for all ids; float32 like the reference's values, written as its float64 column dtype
        table = torch.stack([c.to(dev) for c in per_id]).float().cpu().numpy().astype(np.float64)
        _fresh_folder(self.folder)
        pd.DataFrame(data=table.T, columns=cols).to_csv(os.path.join(self.folder, "distance.csv"), index=False)
        self.stats = {}


def sample_angles_cpu(x):
    """ops.sample_angles for a CPU tensor: the float64 Gram matrix X X^T, cos = G_ij / sqrt(G_ii * G_jj) clamped to
    [-1, 1], NaN where it is not finite, acos in float64 rounded once to float32; 0 on and below the diagonal."""
    t = x.reshape(x.shape[0], -1).double()
    g = t @ t.T
    d = g.diagonal()
    dd = d[:, None] * d[None, :]
    c = g / dd.sqrt()
    ok = torch.isfinite(g) & torch.isfinite(dd) & torch.isfinite(c)
    ang = torch.where(ok, torch.acos(c.clamp(-1.0, 1.0)), torch.full_like(c, float("nan"))).float()
    return torch.triu(ang, diagonal=1)


class AngleStatistics(object):
    """Pairwise angles between the samples of every measured tensor (angle_stats.py:22-80): ``save_measure(t, id)`` records
    the [N, N] matrix acos(cos_sim(t[i], t[j])) for j > i (0 on and below the diagonal); ``__exit__`` stacks each id's
    matrices in call order and pickles {id: DataFrame, ..., 'target': labels} with the ids in first-call order.

    Differences from the reference: the cosine is float64 (from the Gram matrix) instead of fp32, rounded once to float32,
    and clamped to [-1, 1], so nearly parallel samples give a small angle where the reference's fp32 cosine can step over 1
    and give NaN.  A zero sample still gives NaN in its pairs (0 / 0), as in the reference."""

    def __init__(self, folder, base_dir=None):
        self.folder = os.path.join(base_dir or default_base_dir(), "angle", folder)
        self.stats = {}   # id -> float32 [N, N] tensors, one per call (device tensors for CUDA inputs)
        self.targets = []

    def save_measure(self, tensor, id):
        t = tensor.detach()
        prev = self.stats.get(id)
        if prev and prev[0].shape[0] != t.shape[0]:
            raise ValueError("angle measurement of %r: %d samples in this call, %d in the earlier ones"
                             % (id, t.shape[0], prev[0].shape[0]))
        # enqueued now: later in-place writes to the tensor come after it in stream order
        a = ops.sample_angles(t) if t.is_cuda else sample_angles_cpu(t)
        self.stats.setdefault(id, []).append(a)

    def save_target(self, target):
        self.targets = np.concatenate([self.targets, target.detach().cpu().numpy()])

    def __enter__(self):
        return self

    def __exit__(self, *args):
        if not self.stats:
            return
        import pandas as pd
        out = {}
        for id, mats in self.stats.items():   # one device-to-host copy per id
            out[id] = pd.DataFrame(data=torch.cat(mats).cpu().numpy().astype(np.float64))
        out["target"] = self.targets
        _fresh_folder(self.folder)
        with open(os.path.join(self.folder, "angle.pkl"), "wb") as f:
            pickle.dump(out, f)
        self.stats = {}


NOISE_COLUMNS = ["eps_norm", "eps_mse", "eps_cos_sim", "eps_ang_dist", "eps_mean", "eps_var", "w_mean", "w_var", "w_norm",
                 "w_size", "x_mean", "x_var", "x_norm", "x_size", "y_mean", "y_var", "y_norm", "y_size", "c_out"]


def _memory_rows(t, like):
    """[N, row_len] of ``t``'s samples in the memory order of ``like``'s (channels-last rows as stored)."""
    if ops.nhwc(like):
        t = t.permute(0, 2, 3, 1)
    return t.reshape(t.shape[0], -1)


def sample_noise_cpu(y, q=None, bias=None, bias_period=0):
    """ops.sample_noise for CPU tensors: the same float64 sums (columns ops.NOISE_SUMS, the first two without ``q``), with
    ``bias`` added to y in fp32 by the same row convention."""
    yr = _memory_rows(y, y)
    if bias is not None:
        i = torch.arange(yr.shape[1])
        yr = yr + bias.float()[i // bias_period if bias_period > 0 else i % -bias_period]
    yd = yr.double()
    cols = [yd.sum(1), (yd * yd).sum(1)]
    if q is not None:
        qd = _memory_rows(q, y).double()
        e = yd - qd
        cols += [qd.sum(1), (qd * qd).sum(1), (yd * qd).sum(1), e.sum(1), (e * e).sum(1)]
    return torch.stack(cols, 1)


def noise_columns(yq, xs, ws, y_size, x_size, w_size, c_out):
    """The NOISE_COLUMNS of measure_statistics.py:19-99 (float64 [rows, 19], rounded once to float32) from float64 sums:
    ``yq`` [rows, 7] (ops.NOISE_SUMS of the output and its quantized form), ``xs`` / ``ws`` [rows, 2] (sum, sum of squares
    of the input / the weight; NaN without a weight) and the per-row sizes.  Variances are population variances,
    E[t^2] - E[t]^2 in float64 (at least 0).  The cosine is clamped to [-1, 1] before arccos; a zero sample gives a NaN
    cosine and an angular distance of 0, as nan_to_num does in the reference."""
    def mean_var_norm(s, s2, n):
        m = s / n
        return m, np.maximum(s2 / n - m * m, 0.0), np.sqrt(s2)

    rows = yq.shape[0]
    y_size, x_size, w_size, c_out = (np.broadcast_to(np.asarray(v, dtype=np.float64), (rows,))
                                     for v in (y_size, x_size, w_size, c_out))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        cos = yq[:, 4] / np.sqrt(yq[:, 1] * yq[:, 3])
        e_mean, e_var, e_norm = mean_var_norm(yq[:, 5], yq[:, 6], y_size)
        cols = [e_norm, yq[:, 6] / y_size, cos, np.nan_to_num(np.arccos(np.clip(cos, -1.0, 1.0))) / np.pi, e_mean, e_var]
        w_mean, w_var, w_norm = mean_var_norm(ws[:, 0], ws[:, 1], w_size)
        cols += [w_mean, w_var, w_norm, w_size]
        x_mean, x_var, x_norm = mean_var_norm(xs[:, 0], xs[:, 1], x_size)
        cols += [x_mean, x_var, x_norm, x_size]
        y_mean, y_var, y_norm = mean_var_norm(yq[:, 0], yq[:, 1], y_size)
        cols += [y_mean, y_var, y_norm, y_size, c_out]
    return np.stack(cols, 1).astype(np.float32).astype(np.float64)


class NoiseStatistics(object):
    """Quantization noise of every measured call site (measure_statistics.py:19-99): ``save_measure(y, y_with_noise, x, w,
    id)`` records, per sample, the error eps = y - y_with_noise (norm, MSE, cosine and angular distance between y and
    y_with_noise, mean, variance) and the mean, variance, norm and size of the input x, the output y and the weight w,
    plus c_out = w.shape[0]; ``__exit__`` writes one CSV per id, columns NOISE_COLUMNS, one row per sample in call order.
    ``bias`` / ``bias_period`` (ops.sample_noise): a convolution bias the quantization launch added to y itself.  ``w``
    None (a BN without affine parameters): the w_* columns are NaN and c_out is y's channel count.  The weight's moments
    are computed on an id's first call and reused.

    The reference leaves the output location unset (its module is never wired up); <base>/noise/<folder>/ beside
    distance/ and angle/ is this project's choice.  Differences from the reference: everything is computed in float64 and
    rounded once to float32 (the reference computes in fp32), and the cosine is clamped to [-1, 1] before arccos, where the
    reference's fp32 cosine can step over 1 and give NaN, which its nan_to_num turns into the same 0."""

    def __init__(self, folder, base_dir=None):
        self.folder = os.path.join(base_dir or default_base_dir(), "noise", folder)
        self.stats = {}     # id -> [(yq sums [N, 7], x sums [N, 2], y_size, x_size)], one per call
        self.weights = {}   # id -> (weight sums [1, 2] or None, w_size, c_out)

    def save_measure(self, y, y_with_noise, x, w, id, bias=None, bias_period=0):
        y, q, x = y.detach(), y_with_noise.detach(), x.detach()
        # enqueued now: later in-place writes to these tensors come after the launches in stream order
        f = ops.sample_noise if y.is_cuda else sample_noise_cpu
        yq = f(y, q, bias, bias_period)
        xs = f(x)
        if id not in self.weights:
            if w is None:
                self.weights[id] = (None, float("nan"), y.shape[1])
            else:
                w = w.detach()
                self.weights[id] = (f(w.reshape(1, -1)), w.numel(), w.shape[0])
        self.stats.setdefault(id, []).append((yq, xs, y[0].numel(), x[0].numel()))

    def __enter__(self):
        return self

    def __exit__(self, *args):
        if not self.stats:
            return
        import pandas as pd
        tables = {}
        for id, calls in self.stats.items():
            wsum, w_size, c_out = self.weights[id]
            parts = [c[0].reshape(-1) for c in calls] + [c[1].reshape(-1) for c in calls]
            if wsum is not None:
                parts.append(wsum.reshape(-1).to(parts[0].device))
            flat = torch.cat(parts).cpu().numpy()   # one device-to-host copy per id
            rows = sum(c[0].shape[0] for c in calls)
            yq = flat[:rows * 7].reshape(rows, 7)
            xs = flat[rows * 7:rows * 9].reshape(rows, 2)
            ws = np.tile(flat[rows * 9:] if wsum is not None else np.full(2, np.nan), (rows, 1))
            n = [c[0].shape[0] for c in calls]
            tables[id] = noise_columns(yq, xs, ws, np.repeat([c[2] for c in calls], n), np.repeat([c[3] for c in calls], n),
                                       w_size, c_out)
        _fresh_folder(self.folder)
        for id, table in tables.items():
            pd.DataFrame(columns=NOISE_COLUMNS, data=table).to_csv(os.path.join(self.folder, "%s.csv" % id), index=False)
        self.stats, self.weights = {}, {}


MSE_MULTIPLIERS = tuple(0.5 + 0.125 * k for k in range(125))   # clipping values 0.5 .. 16 times b (or std)


def best_columns(multipliers, mse):
    """Per row of ``mse`` ([G, K], one column per multiplier) the column of the smallest MSE; ties go to the smaller
    multiplier and NaN never wins (a row of NaN gives the smallest multiplier)."""
    order = np.argsort(np.asarray(multipliers, dtype=np.float32), kind="stable")
    e = np.asarray(mse, dtype=np.float64)[:, order]
    e = np.where(np.isnan(e), np.inf, e)
    return order[np.argmin(e, axis=1)]


def best_multipliers(multipliers, mse):
    """Per row of ``mse`` ([G, K], one column per multiplier) the multiplier of the smallest MSE (``best_columns``)."""
    return np.asarray(multipliers, dtype=np.float32)[best_columns(multipliers, mse)]


class MseCandidates(object):
    """The clipping candidates of one measurement: the float32 ``multipliers`` and their ``prior`` (ops.clip_mse's:
    alpha = m * b for "laplace", m * std for "gaus"), with one device copy per device.  A manager builds one set from
    mse_multipliers / mse_prior (``of``) and shares it between every measurement of the run."""

    def __init__(self, multipliers, prior):
        self.multipliers = np.asarray(multipliers, dtype=np.float32).reshape(-1)
        self.prior = prior
        self._mult = {}

    @classmethod
    def of(cls, multipliers=None, prior="laplace"):
        """``multipliers`` itself when it is an MseCandidates (a run's shared set), else the candidates of the options
        mse_multipliers (default MSE_MULTIPLIERS) and mse_prior, after checking both."""
        if isinstance(multipliers, cls):
            return multipliers
        if prior not in ("gaus", "laplace"):
            raise ValueError("mse_prior must be one of ['gaus', 'laplace'], got %r" % (prior,))
        cand = cls(MSE_MULTIPLIERS if multipliers is None else multipliers, prior)
        if not 1 <= cand.multipliers.size <= 256:
            raise ValueError("mse_multipliers: 1..256 values, got %d" % cand.multipliers.size)
        return cand

    def mult(self, dev):
        m = self._mult.get(dev)
        if m is None:
            m = torch.from_numpy(self.multipliers)
            if torch.device(dev).type == "cuda":   # pinned and asynchronous: no host synchronisation in a forward
                m = m.pin_memory().to(dev, non_blocking=True)
            self._mult[dev] = m
        return m


class _CallSiteSums(object):
    """The collect and use halves ClipMseStatistics and BitMseStatistics share: per call site, device sums of one launch
    per batch (``_add``), which ``__exit__`` reads back in one copy and writes as ``_tables`` makes them; with ``load``,
    the pickle, read on first use (``_entry``).  Errors name the collect flag FLAG and the use-mode option USE."""

    def __init__(self, folder, base_dir, load):
        self.folder = os.path.join(base_dir or default_base_dir(), self.KIND, folder)
        self.load = load
        self.acc = {}    # id -> (sums [G, n], scales [G, s], float64 device tensors, batches)
        self.meta = {}   # id -> (internal_name, what _tables needs of the call site, elements per group and batch)
        self._loaded = None

    @property
    def path(self):
        return os.path.join(self.folder, self.FILE)

    # -- collect ---------------------------------------------------------------------------------------------------
    def _add(self, id, sums, scales, meta):
        prev = self.acc.get(id)
        if prev is None:
            self.acc[id] = (sums, scales, 1)
            self.meta[id] = meta
            return
        if prev[0].shape != sums.shape:
            raise ValueError("%s of %r: %d %s in this call, %d before" % (self.FLAG, id, sums.shape[0], self.GROUPS,
                                                                          prev[0].shape[0]))
        self.acc[id] = (prev[0] + sums, prev[1] + scales, prev[2] + 1)

    def _read_back(self):
        """(id, sums, batch-mean scales, element count per group, internal name, meta) per call site, from one copy."""
        flat = torch.cat([torch.cat([a[0].reshape(-1), a[1].reshape(-1)]) for a in self.acc.values()]).cpu().numpy()
        pos = 0
        for id, (sums, scales, batches) in self.acc.items():
            g, n = sums.shape
            s = flat[pos:pos + g * n].reshape(g, n)
            pos += g * n
            k = scales.shape[1]
            sc = flat[pos:pos + g * k].reshape(g, k) / batches
            pos += g * k
            tag, info, per_batch = self.meta[id]
            yield id, s, sc, np.full(g, float(per_batch * batches)), tag, info

    def __enter__(self):
        return self

    def __exit__(self, *args):
        if self.load or not self.acc:
            return
        out, csv = self._tables(self._read_back())
        _fresh_folder(self.folder)
        with open(self.path, "wb") as f:
            pickle.dump(out, f)
        csv.to_csv(os.path.join(self.folder, self.CSV), index=False)
        self.acc, self.meta = {}, {}

    # -- use -------------------------------------------------------------------------------------------------------
    def _entry(self, id):
        """The pickle's DataFrame of ``id`` (the pickle is read on first use); KeyError naming FLAG when there is none."""
        if self._loaded is None:
            if not os.path.exists(self.path):
                raise KeyError("%s needs the %ss at %s: collect them with %s=True" % (self.USE, self.WHAT, self.path,
                                                                                      self.FLAG))
            with open(self.path, "rb") as f:
                self._loaded = pickle.load(f)
        df = self._loaded.get(id)
        if df is None:
            raise KeyError("%s needs the %s of layer %r: collect it with %s=True" % (self.USE, self.WHAT, id, self.FLAG))
        return df


class ClipMseStatistics(_CallSiteSums):
    """Clipping-MSE curves (`collect_mse`): ``save_curve(t, tag, id, cfg)`` adds, per group of the quantizer ``cfg`` (a
    ClipErrConfig, as collect_err passes) describes, the float64 sums of its curve (``_curve``) over ``multipliers``
    (alpha = m * b with prior "laplace", m * std with "gaus"; or the run's MseCandidates) and the group's b, std and width
    to device accumulators; ``__exit__`` writes clip_mse.pkl and curve.csv.  With ``load`` the instance reads clip_mse.pkl
    instead (on first use), for `-c mse`.

    curve.csv holds layer totals per element: mse = sum_g sum (x - q)^2 / sum_g count, and the reference's analytic
    curves (mse_analysis.py) per group at the same alpha, with that group's b or std and width (width + 1 for a positive
    range, the relation the reference's *_positive ACIQ tables encode), weighted by the group's count."""
    KIND, FILE, CSV = "clip_mse", "clip_mse.pkl", "curve.csv"
    FLAG, USE, WHAT, GROUPS = "collect_mse", "-c mse", "clipping-MSE curve", "groups"

    def __init__(self, folder, multipliers=None, prior="laplace", base_dir=None, load=False):
        self.candidates = MseCandidates.of(multipliers, prior)
        self.multipliers, self.prior = self.candidates.multipliers, self.candidates.prior
        super(ClipMseStatistics, self).__init__(folder, base_dir, load)

    # -- collect ---------------------------------------------------------------------------------------------------
    def save_curve(self, tensor, tag, id, cfg):
        _, layout, _, table, sums = _curve(tensor.detach(), cfg, self.candidates)
        bits = table[:, 7] if cfg.bit_alloc else torch.full_like(table[:, 7], float(cfg.num_bits))
        self._add(id, sums, torch.stack([table[:, 3], table[:, 4], bits], 1).double(),
                  (tag, bool(cfg.positive), layout[0] * layout[2]))

    def _tables(self, groups):
        import pandas as pd
        from . import mse_analysis
        k = self.multipliers.size
        mults = self.multipliers.astype(np.float64)
        out = {"multipliers": mults, "prior": self.prior}
        rows = []
        for id, s, sc, count, tag, positive in groups:
            g = s.shape[0]
            mse = s[:, 1:] / count[:, None]
            df = pd.DataFrame({"count": count, "b": sc[:, 0], "std": sc[:, 1], "bits": sc[:, 2]})
            out[id] = pd.concat([df, pd.DataFrame(mse, columns=["mse_%d" % j for j in range(k)])], axis=1)
            width = sc[:, 2] + (1 if positive else 0)
            scale = sc[:, 0] if self.prior == "laplace" else sc[:, 1]
            lap = np.empty((g, k))
            gau = np.empty((g, k))
            for r in range(g):
                alpha = mults * scale[r]
                lap[r] = mse_analysis.LaplacianClippingAnalysis(alpha, float(sc[r, 0]), float(width[r])).numpy()
                gau[r] = mse_analysis.GaussianClippingAnalysis(alpha, float(sc[r, 1]), float(width[r])).numpy()
            total = count.sum()
            layer = s[:, 1:].sum(0) / total
            with np.errstate(invalid="ignore", divide="ignore"):
                lap_t = (count[:, None] * lap).sum(0) / total
                gau_t = (count[:, None] * gau).sum(0) / total
            for j in range(k):
                rows.append((id, tag, mults[j], layer[j], lap_t[j], gau_t[j]))
        return out, pd.DataFrame(rows, columns=["id", "internal_name", "multiplier", "mse", "mse_laplace_analytic",
                                                "mse_gaus_analytic"])

    # -- use (`-c mse`) ----------------------------------------------------------------------------------------------
    def best(self, id):
        """(m* per group as float32 [G], prior) of the curve collected for ``id``; KeyError naming collect_mse when there
        is none."""
        df = self._entry(id)
        m = self._loaded["multipliers"]
        return best_multipliers(m, df[["mse_%d" % j for j in range(len(m))]].to_numpy()), self._loaded["prior"]


# The clipping rules a bit-allocation table is measured under (`collect_bits`) and `-bap mse` allocates from: the first
# three with the width candidates of ``bit_candidates``; "mse" (`-c mse`) over a grid of widths and multipliers.
BIT_RULES = ("laplace", "gaus", "no", "mse")


def refuse_bap_mse(kld=False, clipping=None, mid_tread=False, needs_use=False, collect=False, widths_alone=False):
    """Raise NotImplementedError where `-bap mse` would otherwise run another allocation in its place: widths under
    ``-kld`` or a ``clipping`` rule no table is measured under (None: not asked), the ``mid_tread`` (-mtq) bins,
    `-baa` without `-sm use` (``needs_use``), `-baa` while ``collect_err`` / ``collect_mse`` measure (``collect``), and
    the width alone under -c mse (``widths_alone``).  The manager calls it with the run's flags, the quantizer on the
    paths that would run the analytic rule."""
    if widths_alone and clipping == "mse":
        raise NotImplementedError("-bap mse under -c mse picks each channel's width together with its clipping value "
                                  "from the joint tables, not the width alone")
    if kld or (clipping is not None and clipping not in BIT_RULES):
        raise NotImplementedError("-bap mse allocates from tables measured under -c %s, not %s"
                                  % (", ".join(BIT_RULES), "-kld" if kld else "-c " + clipping))
    if mid_tread:
        raise NotImplementedError("-bap mse does not allocate the mid-tread (-mtq) bins")
    if needs_use:
        raise NotImplementedError("-baa -bap mse allocates from per-channel error tables collected with "
                                  "collect_bits=True: it needs -sm use")
    if collect:
        raise NotImplementedError("-baa -bap mse: collect_err and collect_mse would measure their candidates at the "
                                  "analytic widths, not at the widths -bap mse runs with")


def bit_candidates(rule, positive, num_bits):
    """(multipliers, ops.clip_mse prior) of the 9 candidates of width w = 0..8: what `-sm use` runs on a channel
    allocated w bits under the clipping ``rule`` - the Laplace ACIQ factor of w on b (int_quantizer.py:236-253), the Gauss
    factor of ``num_bits`` on std for every width (:264), or the min/max range (:409-451, :453-476)."""
    from .int_quantizer import ALPHA_GAUS, ALPHA_GAUS_POSITIVE, ALPHA_LAPLACE, ALPHA_LAPLACE_POSITIVE
    widths = range(9)
    if rule == "laplace":
        table = ALPHA_LAPLACE_POSITIVE if positive else ALPHA_LAPLACE
        return [table[w] for w in widths], "laplace"
    if rule == "gaus":
        return [(ALPHA_GAUS_POSITIVE if positive else ALPHA_GAUS)[num_bits]] * 9, "gaus"
    if rule == "no":
        return [0.0] * 9, "minmax"
    raise ValueError("bit allocation tables are measured under clipping %s, got %r" % (list(BIT_RULES[:3]), rule))


@functools.lru_cache(maxsize=None)
def _width_candidates(rule, positive, num_bits):
    """The MseCandidates of ``bit_candidates(rule, positive, num_bits)``: constants, made once per key."""
    return MseCandidates(*bit_candidates(rule, positive, num_bits))


class BitMseStatistics(_CallSiteSums):
    """Per-channel error tables of bit allocation (`collect_bits`): ``save_table(t, tag, id, cfg)`` adds, for a call site
    whose quantizer ``cfg`` (a ClipErrConfig) quantizes per channel with bit allocation, the float64 sums of its width
    tables (``_width_tables``: one ops.clip_mse launch over the 9 candidates of ``bit_candidates(rule, ...)``) and the
    channels' b and std to device accumulators; other call sites are skipped.  Under rule "mse" (`-c mse`, the joint
    width-and-clip search) the launch is one ops.clip_mse_grid over widths 0..8 times ``multipliers`` (alpha = m * b with
    ``prior`` "laplace", m * std with "gaus"; or the run's MseCandidates), and each width's error is the one at its best
    multiplier (``best_columns``).  ``__exit__`` writes bit_mse.pkl and alloc.csv.  With ``load`` the instance reads
    bit_mse.pkl instead (on first use), for `-bap mse`."""
    KIND, FILE, CSV = "bit_mse", "bit_mse.pkl", "alloc.csv"
    FLAG, USE, WHAT, GROUPS = "collect_bits", "-bap mse", "per-channel error table", "channels"

    def __init__(self, folder, rule=None, base_dir=None, load=False, multipliers=None, prior="laplace"):
        if not load and rule not in BIT_RULES:
            raise ValueError("collect_bits measures under clipping %s, got %r" % (list(BIT_RULES), rule))
        self.rule = rule
        self.candidates = None
        if rule == "mse":
            self.candidates = MseCandidates.of(multipliers, prior)
            self.multipliers, self.prior = self.candidates.multipliers, self.candidates.prior
        super(BitMseStatistics, self).__init__(folder, base_dir, load)

    # -- collect ---------------------------------------------------------------------------------------------------
    def save_table(self, tensor, tag, id, cfg):
        if not (cfg.per_channel and cfg.bit_alloc):
            return
        _, layout, _, table, sums = _width_tables(tensor.detach(), cfg, self.rule, self.candidates)
        self._add(id, sums, table[:, 3:5].double(), (tag, cfg, layout[0] * layout[2]))

    def _tables(self, groups):
        import pandas as pd
        from . import _lib as L
        from .bit_alloc import allocate
        from .int_quantizer import IntQuantizer
        out = {"rule": self.rule}
        joint = self.rule == "mse"
        if joint:
            out.update(multipliers=self.multipliers.astype(np.float64), prior=self.prior)
        rows = []
        for id, s, sc, count, tag, cfg in groups:
            g = s.shape[0]
            df = pd.DataFrame({"count": count, "b": sc[:, 0], "std": sc[:, 1], "positive": np.full(g, bool(cfg.positive))})
            if joint:   # each width's sum at its best multiplier
                grid = s[:, 1:].reshape(g, 9, -1)
                best = np.stack([best_columns(self.multipliers, grid[:, w]) for w in range(9)], 1)
                sse = np.take_along_axis(grid, best[:, :, None], 2)[:, :, 0]
            else:
                sse = s[:, 1:]
            mse = sse / count[:, None]
            cols = [df, pd.DataFrame(mse, columns=["mse_w%d" % w for w in range(9)])]
            if joint:
                cols.append(pd.DataFrame(self.multipliers[best], columns=["m_w%d" % w for w in range(9)]))
            out[id] = pd.concat(cols, axis=1)
            prior = sc[:, 0] if cfg.bit_alloc_prior == L.PRIOR_B else sc[:, 1]
            analytic = IntQuantizer.get_bits_alloc_fixed_target(torch.from_numpy(prior.astype(np.float32)),
                                                                cfg.bit_alloc_target, cfg.bit_alloc_round)
            allocations = (np.full(g, cfg.num_bits), analytic.numpy().astype(np.int64), allocate(mse, cfg.bit_alloc_target))
            row = [id, tag, g, cfg.bit_alloc_target]
            for w in allocations:
                row += [int(w.sum()), float(sse[np.arange(g), w].sum() / count.sum())]
            rows.append(row)
        return out, pd.DataFrame(rows, columns=ALLOC_COLUMNS)

    # -- use (`-bap mse`) --------------------------------------------------------------------------------------------
    def table(self, id):
        """(float64 [C, 9] per-element MSE of widths 0..8, rule) collected for ``id``; KeyError naming collect_bits when
        there is none."""
        df = self._entry(id)
        return df[["mse_w%d" % w for w in range(9)]].to_numpy(dtype=np.float64), self._loaded["rule"]

    def multipliers_of(self, id):
        """(float32 [C, 9] best multiplier of each width, prior) of a joint table (rule "mse") collected for ``id``."""
        df = self._entry(id)
        return df[["m_w%d" % w for w in range(9)]].to_numpy(dtype=np.float32), self._loaded["prior"]


ALLOC_COLUMNS = ["id", "internal_name", "groups", "target", "bits_uniform", "mse_uniform", "bits_analytic", "mse_analytic",
                 "bits_measured", "mse_measured"]
