"""CPU restatement of measured weight clipping (`clip_weight="mse"`, IntQuantizer._clip_mse_weights), written from the
rule in float64 numpy and the fp32 torch leaf of oracle/fq_oracle.py.  Test infrastructure: the product never imports it.

Per output channel (row) of a weight [O, ...] read as [O, K]:
  1. statistics, float64: min, max, mean, Laplace b = mean |x - mean|, unbiased std (NaN for K = 1);
  2. candidates, from a [O, 12] statistics table (columns _lib.STAT_COLUMNS): column 0 the min/max range (offset = min,
     delta = max - min), then per multiplier m alpha = fp32(m) * fp32(b, or std with the "gaus" prior) as one fp32
     multiply, through fq_oracle.alpha_to_delta_offset in fp32: offset = max(min, mean - alpha), delta = (offset + 2 alpha)
     - offset (the reference forms max_ = offset + range and hands the leaf max_ - offset);
  3. errors: every candidate through fq_oracle.gemmlowp_quantize1 (fp32) at every width in play - num_bits, or 0..8 with
     -baw - and sum (x - q)^2 in float64;
  4. selection: per row and width the first minimum in column order, so min/max wins exact ties and then the earlier
     multiplier; NaN never wins (a row of NaN keeps min/max);
  5. widths: num_bits; with -baw (num_bits <= 4) the table's column 7 (the std prior's widths, restated by std_widths), or
     under -bap mse bit_alloc.allocate on the float64 per-width best errors;
  6. output: the chosen candidate through gemmlowp_quantize1, then fq_oracle.weight_correction (-bcw / -vcw);
  7. the report row of WeightMse.REPORT_COLUMNS: sums over the rows, the errors divided by the element count.

Two tiers: ``row_stats`` is the float64 statistics a table should hold within rounding (tier b); ``restate`` takes the
kernel's own table, so everything it derives must match the device exactly, sums to float64 rounding (tier a).
"""
import numpy as np
import torch

from oracle import fq_oracle as O

CHUNK = 1 << 25   # candidate elements per torch pass


def rows_of(w):
    """float32 [O, K] numpy copy of a weight in NCHW order."""
    w = w.detach().cpu().contiguous() if isinstance(w, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(w))
    return w.reshape(w.shape[0], -1).numpy().astype(np.float32)


def row_stats(w):
    """float64 [O, 5]: min, max, mean, b, std of every row."""
    x = rows_of(w).astype(np.float64)
    with np.errstate(all="ignore"):
        mean = x.mean(1)
        d = x - mean[:, None]
        return np.stack([x.min(1), x.max(1), mean, np.abs(d).mean(1), np.sqrt((d * d).sum(1) / (x.shape[1] - 1))], 1)


def candidates(table, mults, prior):
    """fp32 (delta, offset), each [O, 1 + M]: column 0 min/max, column 1 + k multiplier k."""
    t = np.asarray(table, dtype=np.float32)
    mn, mx, mean = t[:, 0:1], t[:, 1:2], t[:, 2:3]
    scale = t[:, 4 if prior == "gaus" else 3][:, None]
    alpha = np.asarray(mults, dtype=np.float32).reshape(1, -1) * scale
    with np.errstate(all="ignore"):
        rng, off = O.alpha_to_delta_offset(alpha, mx, mn, mean, False)
        delta = (off + rng) - off
    return np.concatenate([mx - mn, delta], 1), np.concatenate([mn, off], 1)


def quantize(x, delta, offset, width):
    """gemmlowp_quantize1 of the rows x [R, K] with per-row delta / offset: ``width`` an int is the num_bits path, an
    array the per-row widths of the bit-allocated path."""
    x, delta, offset = (torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)) for v in (x, delta, offset))
    if isinstance(width, (int, np.integer)):
        return O.gemmlowp_quantize1(x, delta, offset, int(width)).numpy()
    return O.gemmlowp_quantize1(x, delta, offset, None, bit_alloc=torch.from_numpy(np.asarray(width, np.float32))).numpy()


def errors(w, delta, offset, widths, allocated):
    """float64 [O, len(widths), C]: sum (x - q)^2 of every candidate (delta / offset [O, C]) at every width;
    ``allocated``: the widths go through the per-row bit_alloc path of the leaf (as under -baw), else num_bits."""
    x = rows_of(w)
    o, k = x.shape
    c = delta.shape[1]
    out = np.empty((o, len(widths), c))
    step = max(1, CHUNK // max(1, k * c))
    for r0 in range(0, o, step):
        xr = x[r0:r0 + step]
        r = xr.shape[0]
        rep = np.repeat(xr, c, axis=0)   # [r * c, k]: row i candidate j at i * c + j
        xd = torch.from_numpy(rep).double()
        for i, wd in enumerate(widths):
            bits = np.full(r * c, wd, np.float32) if allocated else int(wd)
            y = torch.from_numpy(quantize(rep, delta[r0:r0 + r].reshape(-1), offset[r0:r0 + r].reshape(-1), bits))
            out[r0:r0 + r, i] = ((xd - y.double()) ** 2).sum(1).numpy().reshape(r, c)
    return out


def select(err):
    """(column, error) of the first minimum along the last axis; NaN never wins, a row of NaN keeps column 0."""
    pick = np.argmin(np.where(np.isnan(err), np.inf, err), -1)
    return pick, np.take_along_axis(err, pick[..., None], -1)[..., 0]


def std_widths(table, target, round_=True):
    """-baw with the std prior (the default weight launch's widths): get_bits_alloc_fixed_target on the table's std."""
    std = torch.from_numpy(np.ascontiguousarray(np.asarray(table, np.float32)[:, 4]))
    return O.get_bits_alloc_fixed_target(std, target, round_).numpy().astype(np.float32)


def restate(w, table, mults, prior, num_bits, baw=False, bap_mse=False, target=None, bcw=False, vcw=False, wi=None):
    """Everything `clip_weight="mse"` computes for weight ``w`` from the kernel's statistics ``table`` (tier a), as a dict:
    delta / offset [O, 1 + M] and err [O, W, 1 + M] of every candidate, widths (the W widths in play), pick / best [O, W],
    wi (width index per row), k (chosen column per row), chosen delta / offset / bits [O], y0 (uncorrected) and y
    (corrected) in w's shape, and report (the report row's columns after id and rows, None where empty).  ``wi``: the width
    index of every row instead of the rule's (an allocation of equal total error found from another table)."""
    from cnn_quantization_b200.bit_alloc import allocate
    table = np.asarray(table, dtype=np.float32)
    alloc = bool(baw and num_bits <= 4)
    target = num_bits if target is None else target
    widths = list(range(9)) if alloc else [num_bits]
    delta, offset = candidates(table, mults, prior)
    err = errors(w, delta, offset, widths, alloc)
    pick, best = select(err)
    g = np.arange(len(table))
    if wi is not None:
        wi = np.asarray(wi, np.int64)
    elif not alloc:
        wi = np.zeros(len(table), np.int64)
    elif bap_mse:
        wi = allocate(best, target)
    else:
        wi = table[:, 7].astype(np.int64)
    k = pick[g, wi]
    bits = np.asarray(widths, np.float32)[wi]
    x = rows_of(w)
    y0 = quantize(x, delta[g, k], offset[g, k], bits if alloc else num_bits)
    wt = torch.from_numpy(x).view(w.shape)
    y = O.weight_correction(wt, torch.from_numpy(y0).view(w.shape), bcw, vcw).numpy()
    n = x.size
    ref_bits = ref_sse = None
    if alloc and bap_mse:   # the min/max-only allocation for the same budget
        wmm = allocate(err[:, :, 0], target)
        ref_bits, ref_sse = int(wmm.sum()), err[g, wmm, 0].sum() / n
    report = dict(bits=int(bits.sum()), mse_minmax=err[g, wi, 0].sum() / n, mse_chosen=best[g, wi].sum() / n,
                  kept_minmax=int((k == 0).sum()), bits_minmax_alloc=ref_bits, mse_minmax_alloc=ref_sse)
    return dict(delta=delta, offset=offset, err=err, widths=widths, pick=pick, best=best, wi=wi, k=k,
                chosen=(delta[g, k], offset[g, k], bits), y0=y0.reshape(w.shape), y=y, report=report)


def table_from_stats(stats, bits=None):
    """A [O, 12] statistics table with the columns the restatement reads (min, max, mean, b, std, and the widths in
    column 7), from [O, 5] statistics rounded to fp32: for hand-made rows."""
    s = np.asarray(stats, dtype=np.float64)
    t = np.zeros((len(s), 12), np.float32)
    t[:, :5] = s.astype(np.float32)
    if bits is not None:
        t[:, 7] = bits
    return t


def near_ties(err, best, rel):
    """[..., C] bool: the columns within ``rel`` relative of their row's best that differ from it (sums of distinct
    candidates added in another order may swap such columns; exact ties do not move)."""
    with np.errstate(all="ignore"):
        close = np.abs(err - best[..., None]) <= rel * np.abs(best[..., None])
    return close & (err != best[..., None])
