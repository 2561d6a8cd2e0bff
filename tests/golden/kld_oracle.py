"""CPU restatement of the KL-divergence calibration (`-kld`; the reference's kld_threshold.py:15-80, called per sample by
statistic_manager.py:80-82), written from the algorithm in numpy with the divergence in float64.  Test infrastructure:
the product never imports it.  tests/golden/make_kld_golden.py pins it against the reference itself (ref_kld.npz).

Per sample row:
  1. th = max(|min|, |max|) in fp32; range (-th, th), widened to (-0.5, 0.5) when th == 0;
  2. edges e_k = float32 of numpy.linspace(lo, hi, num_bins + 1) evaluated in float64 (numpy 1.x); h_k = #{e_k <= x < e_{k+1}},
     the last bin closed;
  3. for every candidate i = num_quantized_bins/2 .. num_bins/2: p = the 2i + 1 bins around the zero bin with the outliers
     added to its ends; q = p's bins merged into num_quantized_bins groups and spread over the non-zero bins of each group
     (the last group's spread stops one bin short, so q[-1] = 0); both smoothed with eps = 1e-4; the divergence
     KL(p || q), NaN when q is all zero (the reference's entropy(p, q) then divides 0 by 0);
  4. np.argmin over the candidates (the first NaN, else the first minimum); threshold = e[num_bins/2 + 1 + i];
  5. the layer's kld_th for a batch is the max over its samples (NaN propagates).
"""
import numpy as np

EPS = 0.0001


def legacy_edges(th, num_bins):
    """float32 edges of numpy 1.x's histogram over (-th, th): linspace in float64, then rounded."""
    lo, hi = -float(th), float(th)
    if lo == hi:
        lo, hi = lo - 0.5, hi + 0.5
    return np.linspace(lo, hi, num_bins + 1).astype(np.float32)


def histogram(x, num_bins=2001):
    """(th, edges, counts) of one sample."""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    th = np.float32(max(abs(x.min()), abs(x.max())))
    e = legacy_edges(th, num_bins)
    xs = np.sort(x)
    below = np.concatenate([np.searchsorted(xs, e[:-1], "left"), np.searchsorted(xs, e[-1:], "right")])
    return th, e, np.diff(below).astype(np.int64)


def _smooth(p):
    zeros = p == 0
    nz, nnz = int(zeros.sum()), int(p.size - zeros.sum())
    eps1 = EPS * float(nz) / float(nnz)
    return np.where(zeros, EPS, p - eps1)


def divergences(h, num_quantized_bins=15):
    """The divergence of every candidate, float64 (NaN where q is all zero)."""
    h = np.asarray(h, dtype=np.int64)
    nb, nq = h.size, num_quantized_bins
    z = nb // 2
    out = np.empty(z + 1 - nq // 2)
    for c, i in enumerate(range(nq // 2, z + 1)):
        s, n = z - i, 2 * i + 1
        sl = h[s:s + n]
        p = sl.astype(np.float64)
        p[0] += h[:s].sum()
        p[-1] += h[s + n:].sum()
        m = n // nq
        q = np.zeros(n)
        for j in range(nq):
            start = j * m
            total = sl[start:start + m].sum() if j < nq - 1 else sl[start:].sum()
            stop = start + m if j < nq - 1 else n - 1
            norm = int((sl[start:stop] != 0).sum())
            if norm:
                q[start:stop] = np.float32(float(total) / float(norm))   # the reference's q array is float32
        q[sl == 0] = 0
        if not q.any():
            out[c] = np.nan
            continue
        ps, qs = _smooth(p), _smooth(q)
        P, Q = ps / ps.sum(), qs / qs.sum()
        out[c] = float(np.sum(P * np.log(P / Q)))
    return out


def search(h, edges, num_quantized_bins=15):
    """(threshold, divergence, index into the candidates) of one sample's histogram."""
    div = divergences(h, num_quantized_bins)
    idx = int(np.argmin(div))
    return edges[len(h) // 2 + 1 + num_quantized_bins // 2 + idx], div[idx], idx


def kld_threshold(x, num_bins=2001, num_quantized_bins=15):
    """Per-sample (th[N], div[N], idx[N]) of x[N, ...]; a sample with NaN / Inf gives (NaN, NaN, -1)."""
    x = np.asarray(x, dtype=np.float32)
    th, dv, ix = [], [], []
    for row in x.reshape(x.shape[0], -1):
        if not np.isfinite(row).all():
            th.append(np.nan), dv.append(np.nan), ix.append(-1)
            continue
        _, e, h = histogram(row, num_bins)
        t, d, i = search(h, e, num_quantized_bins)
        th.append(t), dv.append(d), ix.append(i)
    return np.asarray(th, dtype=np.float32), np.asarray(dv), np.asarray(ix, dtype=np.int32)


# ---- the fixture rows (tests/golden/ref_kld.npz stores kind, shape and seed; the data is regenerated from them) --------
SHAPES = ((64, 56, 56), (256, 14, 14), (2048, 7, 7))   # ResNet-50 per-sample activations


def make_row(kind, shape, seed):
    rs = np.random.RandomState(seed)
    if kind == "normal":
        return rs.standard_normal(shape).astype(np.float32)
    if kind == "laplace":
        return rs.laplace(size=shape).astype(np.float32)
    if kind == "relu":
        return np.maximum(rs.standard_normal(shape), 0).astype(np.float32)
    if kind == "outlier":
        x = rs.standard_normal(shape).astype(np.float32)
        x.reshape(-1)[rs.randint(x.size)] = 60.0
        return x
    if kind == "zeros":
        return np.zeros(shape, np.float32)
    if kind == "const2":
        return np.full(shape, 2.0, np.float32)
    if kind == "single":
        x = np.zeros(shape, np.float32)
        x.reshape(-1)[rs.randint(x.size)] = 1.5
        return x
    if kind == "positive":   # all mass far from zero: the small candidates see an all-zero q (NaN)
        return (3.0 + rs.rand(*shape)).astype(np.float32)
    raise ValueError(kind)


def fixture_rows():
    """[(kind, shape, seed)] of ref_kld.npz."""
    rows, seed = [], 100
    for kind in ("normal", "laplace", "relu", "outlier"):
        for shape in SHAPES:
            rows.append((kind, shape, seed))
            seed += 1
    for kind in ("zeros", "const2", "single", "positive"):
        rows.append((kind, (256, 14, 14), seed))
        seed += 1
    return rows
