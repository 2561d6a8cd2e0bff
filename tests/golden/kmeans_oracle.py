"""Float64 numpy restatement of the 1-D k-means of ``ops.kmeans1d`` (csrc/fq_kmeans.cuh), with the same random draws and the
same summation orders where they decide a discrete choice (the k-means++ potentials and cumulative sums, the mean, the
variance, the inertia).  It follows scikit-learn 1.9's ``KMeans(n_clusters=k, random_state=seed).fit`` (``fit``,
``_kmeans_plusplus``, ``_tolerance``, ``_kmeans_single_lloyd``, ``_relocate_empty_clusters_dense``) in float64; the only
rules it adds are the ones scikit-learn leaves to its BLAS / argpartition:

- sums: blocks of 512 elements (16 rows of 32 lanes, each lane adds its column in order, then an xor butterfly over the 32
  lanes), superblocks of 32 blocks (the same butterfly), superblocks added one after the other;
- searchsorted(cumsum, v, 'left'): the first superblock whose running total reaches v, then the first block of it whose
  running total (from the superblock's start) does, then the first element of that block (the last block / element when
  rounding leaves none; n - 1 when no superblock reaches v);
- relocation of empty clusters: the farthest points first, ties to the lowest index;
- convergence shift: the sum over clusters of (c_new - c_old)^2 in cluster order.
Per-cluster sums of the Lloyd update are plain numpy sums (the device's order differs in the last bits).  Test
infrastructure, like kld_oracle.py."""
import numpy as np

BLK, ROWS, SUPER, MAX_ITER, TOL = 512, 16, 32, 300, 1e-4
_PERM = [np.arange(32) ^ o for o in (16, 8, 4, 2, 1)]


def _butterfly(a):
    for p in _PERM:
        a = a + a[:, p]
    return a[:, 0]


def hsum(d):
    """(per-block sums, per-superblock sums, total) of a float64 vector in the device's order."""
    n = d.size
    nb = -(-n // BLK)
    nsb = -(-nb // SUPER)
    pad = np.zeros(nb * BLK)
    pad[:n] = d
    d3 = pad.reshape(nb, ROWS, 32)
    acc = np.zeros((nb, 32))
    for r in range(ROWS):
        acc = acc + d3[:, r, :]
    blk = _butterfly(acc)
    padb = np.zeros(nsb * SUPER)
    padb[:nb] = blk
    sup = _butterfly(padb.reshape(nsb, SUPER))
    return blk, sup, float(np.cumsum(sup)[-1])


def search(d, blk, sup, v):
    """searchsorted(cumsum(d), v, side='left') clipped to n - 1, with the cumulative sum of the hierarchy."""
    n = d.size
    cs = np.cumsum(sup)
    hit = np.nonzero(cs >= v)[0]
    if hit.size == 0:
        return n - 1
    g = int(hit[0])
    q = float(cs[g - 1]) if g else 0.0
    b0, b1 = g * SUPER, min(g * SUPER + SUPER, blk.size)
    rs = np.cumsum(np.concatenate([[q], blk[b0:b1]]))
    hit = np.nonzero(rs[1:] >= v)[0]
    b = b0 + (int(hit[0]) if hit.size else b1 - 1 - b0)
    r = float(rs[b - b0])
    e0, e1 = b * BLK, min(b * BLK + BLK, n)
    es = np.cumsum(np.concatenate([[r], d[e0:e1]]))
    hit = np.nonzero(es[1:] >= v)[0]
    return e0 + (int(hit[0]) if hit.size else e1 - 1 - e0)


def synthetic(kind, n, seed):
    """The synthetic fixture tensors: Gaussian, Laplace, Gaussian with 0.1 % outliers at 80x, and a tensor of 9 distinct
    values (fewer than k at 4 bits: the empty-cluster path)."""
    rng = np.random.RandomState(seed)
    if kind == "gauss":
        return (rng.randn(n) * 0.05).astype(np.float32)
    if kind == "laplace":
        return rng.laplace(0.0, 0.02, n).astype(np.float32)
    if kind == "outliers":
        x = rng.randn(n) * 0.01
        x[rng.choice(n, n // 1000, replace=False)] *= 80.0
        return x.astype(np.float32)
    assert kind == "few"
    return np.repeat(np.linspace(-1.0, 1.0, 9), -(-n // 9))[:n].astype(np.float32)


# synthetic fixtures: name -> (kind, n, seed, num_bits)
SYNTHETIC = {"gauss": ("gauss", 200000, 1, 4), "laplace": ("laplace", 200000, 2, 4), "outliers": ("outliers", 200000, 3, 4),
             "few": ("few", 4000, 4, 4), "mid_2bit": ("laplace", 147456, 5, 2), "mid_8bit": ("laplace", 147456, 5, 8)}


def far_centres_case():
    """(x, init) of a relocation case on continuous data: 5000 Gaussian values and 16 initial centres, three of them far
    away, so three clusters are empty at the first iteration and take the farthest points."""
    x = (np.random.RandomState(11).randn(5000) * 0.1).astype(np.float32)
    return x, np.concatenate([[-50.0, 40.0, -30.0], np.linspace(-0.2, 0.2, 13)])


def sample_positions(n):
    """The positions whose labels the fixtures keep: all of them up to 65536, else a seeded sample of 65536."""
    if n <= 65536:
        return np.arange(n)
    return np.sort(np.random.RandomState(7).choice(n, 65536, replace=False))


def n_trials(k):
    return 2 + int(np.log(k))


def draws(n, k, seed):
    """scikit-learn's k-means++ draws on RandomState(seed): choice(n, p=w / w.sum()) with float32 unit weights, then
    uniform(size=n_local_trials) per further centre."""
    rs = np.random.RandomState(seed)
    w = np.ones(n, dtype=np.float32)
    first = int(rs.choice(n, p=w / w.sum()))
    t = n_trials(k)
    return first, np.array([rs.uniform(size=t) for _ in range(k - 1)]).reshape(k - 1, t)


def assign(xc, c, chunk=1 << 16):
    """np.argmin over the centres of (x - c)^2: the nearest centre, ties to the lowest index."""
    out = np.empty(xc.size, dtype=np.int64)
    for i in range(0, xc.size, chunk):
        out[i:i + chunk] = np.argmin((xc[i:i + chunk, None] - c[None, :]) ** 2, axis=1)
    return out


def kmeans_pp(xc, k, seed):
    """(centred centres, sample indices) of k-means++."""
    first, u = draws(xc.size, k, seed)
    d = np.full(xc.size, np.inf)
    cand, centres, ids = [first], [], []
    for c in range(k):
        cols = [np.minimum(d, (xc - xc[i]) ** 2) for i in cand]
        sums = [hsum(col) for col in cols]
        best = int(np.argmin([s[2] for s in sums]))
        centres.append(xc[cand[best]])
        ids.append(cand[best])
        d = cols[best]
        if c + 1 < k:
            blk, sup, pot = sums[best]
            cand = [search(d, blk, sup, float(ut * pot)) for ut in u[c]]
    return np.array(centres), np.array(ids)


def kmeans(x, num_bits, seed=0, init=None, task=None, rows=None):
    """dict(labels, centres (float32), centres64 (centred), inertia, n_iter, init_ids, init64 (centred), out, out_bcorr)."""
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
    k = 1 << num_bits
    n = x.size
    assert n >= k
    xd = x.astype(np.float64)
    mean = hsum(xd)[2] / n
    xc = xd - mean
    tol = hsum(xc * xc)[2] / n * TOL
    if init is None:
        c, ids = kmeans_pp(xc, k, seed)
    else:
        c, ids = np.asarray(init, dtype=np.float64).reshape(-1) - mean, np.full(k, -1)
    c_init = c.copy()
    relocated = 0
    strict = False
    labels_old = None
    for it in range(MAX_ITER):
        labels = assign(xc, c)
        sums = np.bincount(labels, weights=xc, minlength=k).astype(np.float64)
        cnt = np.bincount(labels, minlength=k).astype(np.int64)
        empty = np.nonzero(cnt == 0)[0]
        if empty.size:
            dist = (xc - c[labels]) ** 2
            if dist.max() > 0:
                far = np.lexsort((np.arange(n), -dist))[:empty.size]
                relocated += empty.size
                for j, f in zip(empty, far):
                    old = labels[f]
                    sums[old] = sums[old] - xc[f]
                    sums[j] = xc[f]
                    cnt[j] = 1
                    cnt[old] -= 1
        amax = int(np.argmax(cnt))
        new = sums.copy()
        for j in range(k):
            new[j] = new[j] * (1.0 / cnt[j]) if cnt[j] > 0 else new[amax]
        shift = 0.0
        for j in range(k):
            shift = shift + (new[j] - c[j]) ** 2
        c = new
        if labels_old is not None and np.array_equal(labels, labels_old):
            strict = True
            break
        if shift <= tol:
            break
        labels_old = labels
    n_iter = it + 1
    if not strict:
        labels = assign(xc, c)
    inertia = hsum((xc - c[labels]) ** 2)[2]
    cf = (c + mean).astype(np.float32)
    out = out_bcorr = None
    if task == "quantize":
        out = cf[labels]
    elif task == "clip":
        out = np.clip(x, cf.min(), cf.max())
    if rows:
        q = out.reshape(rows, -1).astype(np.float64)
        w = xd.reshape(rows, -1)
        delta = q.mean(1) - w.mean(1)
        out_bcorr = (q - delta[:, None]).astype(np.float32).reshape(-1)
    return dict(labels=labels, centres=cf, centres64=c, inertia=inertia, n_iter=n_iter, init_ids=ids, init64=c_init,
                mean=mean, out=out, out_bcorr=out_bcorr, strict=strict, relocated=relocated)
