"""CPU tests of the 1-D k-means quantization: the C ABI's argument checks and workspace sizes, the float64 restatement
(tests/golden/kmeans_oracle.py) against scikit-learn's runs of the reference script (tests/golden/kmeans_ref.npz, tiers
in kmeans_tiers.py), the reference's is_ignored decisions, process_model's file names, the bias-correction formula on the
reference's own quantized tensor, and that CPU tensors raise.  The two comparisons with a live scikit-learn fit skip
where scikit-learn is not installed; the fixtures carry everything else."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLDEN)
import kmeans_oracle as KO  # noqa: E402
import kmeans_tiers as KT  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLDEN, "kmeans_ref.npz"))


def test_workspace_bytes(lib):
    from cnn_quantization_b200 import _lib
    for n, k in ((16, 16), (1000, 2), (2359296, 16), (102760448, 16), (147456, 256)):
        assert lib.fqb200_kmeans1d_workspace_bytes(n, k) > 0
    assert lib.fqb200_kmeans1d_workspace_bytes(2359296, 256) > lib.fqb200_kmeans1d_workspace_bytes(2359296, 16)
    for n, k in ((15, 16), (100, 3), (100, 1), (100, 512), (1 << 40, 16)):
        assert lib.fqb200_kmeans1d_workspace_bytes(n, k) == 0
        assert lib.fqb200_last_error()
    assert _lib.ERR_INVALID == 1


def test_argument_errors(lib):
    from cnn_quantization_b200 import _lib
    fake = 1 << 20   # never dereferenced: every check below fails before any device work
    ws = lib.fqb200_kmeans1d_workspace_bytes(1000, 16)

    def call(**over):
        a = dict(inp=fake, n=1000, bits=4, first=0, draws=fake, trials=4, init=None, task=1, rows=0, labels=fake,
                 centres=fake, inertia=fake, n_iter=fake, ids=fake, out=fake, bcorr=None, ws=fake, wsb=ws, max_ctas=0)
        a.update(over)
        return lib.fqb200_kmeans1d(a["inp"], a["n"], a["bits"], a["first"], a["draws"], a["trials"], a["init"], a["task"],
                                   a["rows"], a["labels"], a["centres"], a["inertia"], a["n_iter"], a["ids"], a["out"],
                                   a["bcorr"], a["ws"], a["wsb"], a["max_ctas"], None)
    bad = [dict(bits=0), dict(bits=9), dict(n=10), dict(inp=None), dict(labels=None), dict(centres=None), dict(task=3),
           dict(out=None), dict(rows=-1), dict(rows=7), dict(rows=10), dict(rows=10, task=0), dict(draws=None),
           dict(first=1000), dict(first=-1), dict(trials=0), dict(trials=8), dict(max_ctas=-1)]
    for over in bad:
        assert call(**over) == _lib.ERR_INVALID, over
    assert call(wsb=ws - 1) == _lib.ERR_WORKSPACE
    assert call(ws=None) == _lib.ERR_WORKSPACE
    assert call(ws=fake + 8) == _lib.ERR_WORKSPACE


def test_cpu_tensor_raises():
    import cnn_quantization_b200 as fq
    with pytest.raises(fq._lib.FqError):
        fq.ops.kmeans1d(torch.randn(1000), 4)


def test_draws_match_numpy():
    import cnn_quantization_b200 as fq
    for n, k, seed in ((1000, 16, 0), (70001, 4, 0), (5000, 256, 3)):
        a, ua = fq.ops.kmeans_draws(n, k, seed)
        b, ub = KO.draws(n, k, seed)
        assert a == b and np.array_equal(ua, ub) and ua.shape == (k - 1, 2 + int(np.log(k)))


def test_restatement_small_matches_scikit_learn():
    """On a small tensor every float32 / float64 difference is too small to move a choice: the restatement reproduces
    scikit-learn's whole fit, k-means++ included."""
    KMeans = pytest.importorskip("sklearn.cluster").KMeans
    x = np.random.RandomState(1).randn(64, 3, 3, 3).astype(np.float32)
    r = KO.kmeans(x, 4, seed=0, task="quantize")
    km = KMeans(n_clusters=16, random_state=0).fit(x.reshape(-1, 1))
    assert r["n_iter"] == km.n_iter_
    assert np.abs(r["centres"] - km.cluster_centers_[:, 0]).max() <= 1e-6
    assert np.array_equal(r["labels"], km.labels_)


def test_restatement_relocation_matches_scikit_learn():
    """Three empty clusters at the first iteration, filled with the farthest points: the restatement follows
    _relocate_empty_clusters_dense and the rest of scikit-learn's run to its float32 rounding."""
    KMeans = pytest.importorskip("sklearn.cluster").KMeans
    x, init = KO.far_centres_case()
    r = KO.kmeans(x, 4, init=init)
    assert r["relocated"] == 3
    km = KMeans(n_clusters=16, init=init.reshape(-1, 1), n_init=1).fit(x.reshape(-1, 1))
    assert r["n_iter"] == km.n_iter_
    assert np.array_equal(r["labels"], km.labels_)
    assert np.abs(r["centres"] - km.cluster_centers_[:, 0]).max() <= 1e-6 * float(x.max() - x.min())


def test_restatement_search_is_searchsorted():
    rng = np.random.RandomState(2)
    d = rng.rand(40000) ** 4
    blk, sup, tot = KO.hsum(d)
    cs = np.cumsum(d)
    for u in rng.rand(200):
        v = u * tot
        i = KO.search(d, blk, sup, v)
        j = min(int(np.searchsorted(cs, v)), d.size - 1)
        assert abs(i - j) <= 1 and abs(cs[i] - v) <= 1e-9 * tot + d[i]


@pytest.mark.parametrize("tier", ["i", "ii"])
def test_restatement_against_reference(ref, tier):
    for name in KT.names(ref):
        if name.startswith("resnet18/layer4") or name.startswith("resnet18/layer3"):
            continue   # the biggest tensors run on the GPU (tests/test_gpu_kmeans.py); here the restatement is slow
        x = KT.fixture_tensor(ref, name)
        bits = int(ref["bits/" + name])
        if tier == "i":
            r = KO.kmeans(x, bits, init=ref["ref_init/" + name])
            KT.check_tier_i(ref, name, x, r["n_iter"], r["centres"], r["labels"], r["inertia"])
        else:
            r = KO.kmeans(x, bits, seed=0)
            KT.check_tier_ii(ref, name, x, r["init_ids"], r["inertia"])


def test_reference_label_counts_and_clip_bounds(ref):
    for name in KT.names(ref):
        c = ref["ref_centres/" + name].astype(np.float32)
        x = KT.fixture_tensor(ref, name)
        assert ref["ref_counts/" + name].sum() == x.size
        if "ref_clip/" + name in ref.files:
            # the clipped tensor's range: the centres' range inside the data's.  clip1d_kmeans fits again, and
            # scikit-learn adds its threads' float32 partial sums in whichever order they finish: a few ulp apart
            lo, hi = ref["ref_clip/" + name]
            tol = 1e-6 * float(x.max() - x.min())
            assert abs(lo - max(c.min(), x.min())) <= tol and abs(hi - min(c.max(), x.max())) <= tol


def test_is_ignored_matches_reference(ref):
    from cnn_quantization_b200.kmeans_quantization import is_ignored

    class P(object):
        def __init__(self, shape):
            self.shape = tuple(int(v) for v in shape if v) or (0,)

    for arch in ("resnet50", "vgg16", "inception_v3"):
        names_ = ref["ignored_names/" + arch]
        shapes = ref["ignored_shapes/" + arch]
        want = ref["ignored/" + arch]
        got = [bool(is_ignored(str(n), P(s))) for n, s in zip(names_, shapes)]
        assert got == [bool(w) for w in want], arch
    # VGG-16's classifier.6.weight (1000 x 4096) has no 'fc' in its name: it is clustered
    vgg = dict(zip((str(n) for n in ref["ignored_names/vgg16"]), ref["ignored/vgg16"]))
    assert not vgg["classifier.6.weight"] and vgg["classifier.6.bias"] and vgg["features.0.weight"]


def test_process_model_paths(ref):
    from cnn_quantization_b200.kmeans_quantization import model_paths
    p, q = model_paths("resnet18", 4, "/tmp/base")
    assert [os.path.basename(p), os.path.basename(q)] == sorted(str(s) for s in ref["saved"])
    # a dot in the directory: the reference's path.split('.')[0] would cut there; the extension is replaced instead
    p, q = model_paths("resnet50", 8, "/data/v1.2/run")
    assert p == "/data/v1.2/run/models/resnet50_kmeans8bit.pt" and q == "/data/v1.2/run/models/resnet50_kmeans8bit_bcorr.pt"


def test_bias_correction_formula_on_reference_tensor(ref):
    """The reference's quantized layer1.0.conv1.weight (its centres at its labels, all 36864 kept) through the float64
    row-mean formula of the kernel gives the reference's bias-corrected tensor to float32 rounding."""
    name = "resnet18/layer1.0.conv1.weight"
    x = KT.fixture_tensor(ref, name)
    wq = ref["ref_centres/" + name].astype(np.float32)[ref["ref_labels/" + name]]
    rows = 64
    q, w = wq.reshape(rows, -1).astype(np.float64), x.reshape(rows, -1).astype(np.float64)
    got = (q - (q.mean(1) - w.mean(1))[:, None]).astype(np.float32).reshape(-1)
    want = ref["ref_bcorr/" + name]
    assert np.abs(got - want).max() <= 4 * np.spacing(np.abs(want).max())
