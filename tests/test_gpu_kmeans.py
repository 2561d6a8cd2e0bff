"""GPU tests of the 1-D k-means quantization (ops.kmeans1d, csrc/fq_kmeans.cuh; kmeans_quantization.py):
- against the float64 restatement tests/golden/kmeans_oracle.py: the same init indices and n_iter, identical labels,
  centres within 1e-12 of their scale, inertia within 1e-12 relative, the written tensor bit for bit where the fp32 centres
  agree;
- the relocation of empty clusters to the farthest points (far-away initial centres; a far point alone in its cluster,
  whose cluster then empties too) against the restatement;
- tier (i), against scikit-learn's own run (tests/golden/kmeans_ref.npz) started from its own init centres, with the
  bounds of tests/golden/kmeans_tiers.py: the same n_iter, centres within 3e-5 of the range, sampled labels equal but for
  a fraction of at most 5e-4 (scikit-learn fits in float32; the measured worst cases are 2.1e-5 and 3.2e-4), and the 8-bit
  tensor, whose float32 and float64 runs stop one iteration apart, on its inertia within 0.5 %;
- tier (ii), end to end against scikit-learn: the first k-means++ pick, and the inertia within 6 % (5.1 % measured);
- determinism over runs and grid sizes, VGG-16 fc6's shape at 4 bits (Lloyd fixed point in float64), the clip task, the
  bias correction, and ResNet-18 end to end."""
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

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fq():
    import __graft_entry__
    __graft_entry__.build()
    import cnn_quantization_b200 as fq
    return fq


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLDEN, "kmeans_ref.npz"))


_synthetic = KO.synthetic


CASES = [("gauss", 60000, 4), ("laplace", 131072, 4), ("outliers", 50000, 4), ("few", 4000, 4), ("gauss", 70001, 2),
         ("laplace", 20000, 8), ("gauss", 2000, 1)]


def _run(fq, x, bits, **kw):
    r = fq.ops.kmeans1d(torch.from_numpy(x).cuda(), bits, **kw)
    torch.cuda.synchronize()
    return r


@pytest.mark.parametrize("kind,n,bits", CASES)
def test_against_restatement(fq, kind, n, bits):
    x = _synthetic(kind, n, n + bits)
    want = KO.kmeans(x, bits, seed=0, task="quantize")
    got = _run(fq, x, bits, seed=0, task="quantize")
    assert got.init_ids.cpu().numpy().tolist() == want["init_ids"].tolist()
    assert int(got.n_iter) == want["n_iter"]
    assert np.array_equal(got.labels.cpu().numpy().astype(np.int64), want["labels"])
    _check_centres_and_out(got, want)


def _check_centres_and_out(got, want):
    """Centres within 1e-12 of their scale (the per-cluster sums are added in another order; a centre at a cancelling
    zero shows it), the inertia within 1e-12 relative, and the written tensor bit for bit: its own centres at the shared
    labels, the restatement's values wherever the fp32 centres agree."""
    c = got.centres.cpu().numpy()
    scale = np.abs(want["centres"]).max()
    assert np.abs(c.astype(np.float64) - want["centres"]).max() <= 1e-12 * scale + np.spacing(np.float32(scale))
    # (a tensor of few distinct values has an inertia of pure rounding noise: bounded by the data's scale)
    assert abs(float(got.inertia) - want["inertia"]) <= 1e-12 * abs(want["inertia"]) + 1e-20 * c.size * scale ** 2
    out = got.out.cpu().numpy().reshape(-1)
    assert np.array_equal(out, c[want["labels"]])
    same = (c == want["centres"])[want["labels"]]
    assert np.array_equal(out[same], want["out"][same])


# 128 values with a sum of a few halves: the mean and every cluster mean are exact in float64, so no tie between equal
# centres is decided by rounding
RELOCATION_CASES = {
    # the farthest point (5.0) is alone in cluster 3: filling empty cluster 0 empties cluster 3 as well
    "singleton_above": (np.r_[np.zeros(63), np.ones(64), 5.0], [-100.0, 0.0, 1.0, 7.0], 2),
    # the same with the far point's cluster below the empty one
    "singleton_below": (np.r_[5.0, np.zeros(63), np.ones(64)], [7.0, -100.0, 0.0, 1.0], 2),
    # four empty clusters; both points of cluster 4 are among the four farthest
    "four_empty": (np.r_[np.zeros(62), np.ones(63), 5.0, 5.5, 9.0], [-100.0, -200.0, 0.0, 1.0, 5.2, 9.0, 300.0, 400.0], 3),
    # three far-away centres on continuous data (scikit-learn's run is the same: tests/test_kmeans_cpu.py)
    "far_centres": KO.far_centres_case() + (4,),
}


@pytest.mark.parametrize("case", sorted(RELOCATION_CASES))
def test_relocation_against_restatement(fq, case):
    x, init, bits = RELOCATION_CASES[case]
    x = np.asarray(x, dtype=np.float32)
    want = KO.kmeans(x, bits, init=init, task="quantize")
    assert want["relocated"] > 0   # the case really moves points (the farthest distance is > 0)
    for max_ctas in (0, 1, 3):
        got = _run(fq, x, bits, init=np.asarray(init), task="quantize", max_ctas=max_ctas)
        assert int(got.n_iter) == want["n_iter"], case
        assert np.array_equal(got.labels.cpu().numpy().astype(np.int64), want["labels"]), case
        _check_centres_and_out(got, want)


def test_clip_and_bias_correction(fq):
    x = (np.random.RandomState(3).randn(64, 32, 3, 3) * 0.1).astype(np.float32)
    want = KO.kmeans(x, 4, seed=0, task="clip")
    got = _run(fq, x, 4, task="clip", rows=64)
    assert np.array_equal(got.out.cpu().numpy().reshape(-1), want["out"])
    lo, hi = want["centres"].min(), want["centres"].max()
    assert float(got.out.min()) >= lo and float(got.out.max()) <= hi
    # bias correction against the torch float64 formula, rounded to fp32 once
    for task in ("clip", "quantize"):
        got = _run(fq, x, 4, task=task, rows=64)
        w, q = torch.from_numpy(x).double().view(64, -1), got.out.cpu().double().view(64, -1)
        expect = (q - (q.mean(1) - w.mean(1)).view(64, 1)).float()
        b = got.out_bcorr.cpu().view(64, -1)
        assert (b - expect).abs().max().item() <= 1e-7 * max(1.0, expect.abs().max().item())
        assert torch.allclose(b.double().mean(1), w.mean(1), rtol=0, atol=1e-6)


def test_given_init_and_determinism(fq):
    x = _synthetic("laplace", 300000, 5)
    init = np.linspace(x.min(), x.max(), 16)
    want = KO.kmeans(x, 4, init=init)
    ref_run = _run(fq, x, 4, init=init, task="quantize")
    assert int(ref_run.n_iter) == want["n_iter"]
    assert (ref_run.init_ids.cpu() == -1).all()
    assert np.array_equal(ref_run.labels.cpu().numpy().astype(np.int64), want["labels"])
    assert np.array_equal(ref_run.centres.cpu().numpy(), want["centres"])
    for max_ctas in (0, 0, 1, 7, 100):
        for kw in (dict(init=init), dict(seed=0)):
            base = _run(fq, x, 4, task="quantize", **kw) if max_ctas == 0 else None
            r = _run(fq, x, 4, task="quantize", max_ctas=max_ctas, **kw)
            other = ref_run if "init" in kw else _run(fq, x, 4, task="quantize", seed=0)
            for a, b in ((r, other),) + (((base, other),) if base is not None else ()):
                assert torch.equal(a.labels, b.labels) and torch.equal(a.centres, b.centres)
                assert torch.equal(a.inertia, b.inertia) and torch.equal(a.out, b.out)
                assert int(a.n_iter) == int(b.n_iter) and torch.equal(a.init_ids, b.init_ids)


def test_errors(fq):
    x = torch.randn(100, device="cuda")
    with pytest.raises(ValueError):
        fq.ops.kmeans1d(x, 7)            # n < k
    y = x.clone()
    y[3] = float("nan")
    with pytest.raises(ValueError):
        fq.ops.kmeans1d(y, 2)
    y[3] = float("inf")
    with pytest.raises(ValueError):
        fq.ops.kmeans1d(y, 2)
    with pytest.raises(ValueError):
        fq.ops.kmeans1d(x, 2, task="clip", rows=7)


def test_vgg16_fc6_shape_fixed_point(fq):
    """25088 x 4096 (VGG-16 classifier.0) at 4 bits: every label is a nearest centre and every centre the mean of its
    points, checked in float64 torch."""
    g = torch.Generator(device="cuda").manual_seed(6)
    w = torch.randn(4096, 25088, device="cuda", generator=g) * 0.01
    r = fq.ops.kmeans1d(w, 4, task="quantize")
    torch.cuda.synchronize()
    assert int(r.n_iter) <= 300
    xd = w.reshape(-1).double()
    c = r.centres.double()
    lab = r.labels.reshape(-1).long()
    # nearest centre (float32 centres: allow the rounding of the centres themselves)
    d_own = (xd - c[lab]).abs()
    cs, _ = torch.sort(c)
    pos = torch.searchsorted(cs, xd).clamp(1, c.numel() - 1)
    d_best = torch.minimum((xd - cs[pos - 1]).abs(), (xd - cs[pos]).abs())
    slack = 2 * torch.finfo(torch.float32).eps * c.abs().max()
    assert bool((d_own <= d_best + slack).all())
    cnt = torch.bincount(lab, minlength=16).double()
    sums = torch.zeros(16, dtype=torch.float64, device="cuda").index_add_(0, lab, xd)
    assert bool((cnt > 0).all())
    means = sums / cnt
    rng = float(xd.max() - xd.min())
    if int(r.n_iter) < 300:
        # converged: centres are the cluster means up to the tolerance of the last shift and fp32 rounding
        assert float((means - c).abs().max()) <= 1e-3 * rng
    assert torch.equal(r.out.reshape(-1), r.centres[lab])


@pytest.mark.parametrize("name", ["resnet18/layer1.0.conv1.weight", "resnet18/layer3.1.conv2.weight",
                                  "resnet18/layer4.1.conv2.weight", "synthetic/few", "synthetic/mid_8bit"])
def test_restatement_fixture_tensors(fq, ref, name):
    """GPU = restatement on the fixtures' tensors (ResNet-18 weights up to 2.36 M elements, the empty-cluster path, 8 bits)."""
    x = KT.fixture_tensor(ref, name)
    bits = int(ref["bits/" + name])
    want = KO.kmeans(x, bits, seed=0, task="quantize")
    got = _run(fq, x, bits, task="quantize")
    assert got.init_ids.cpu().numpy().tolist() == want["init_ids"].tolist()
    assert int(got.n_iter) == want["n_iter"]
    assert np.array_equal(got.labels.cpu().numpy().reshape(-1).astype(np.int64), want["labels"])
    _check_centres_and_out(got, want)


def test_tier_i_given_reference_init(fq, ref):
    """Started from scikit-learn's own init centres, the GPU follows its Lloyd run (bounds: kmeans_tiers.py)."""
    for name in KT.names(ref):
        x = KT.fixture_tensor(ref, name)
        r = _run(fq, x, int(ref["bits/" + name]), init=ref["ref_init/" + name], task="quantize")
        KT.check_tier_i(ref, name, x, int(r.n_iter), r.centres.cpu().numpy(), r.labels.cpu().numpy().reshape(-1),
                        float(r.inertia))


def test_tier_ii_end_to_end(fq, ref):
    """k-means++ on the GPU against scikit-learn's whole run: the first pick, and the inertia within the measured bound."""
    for name in KT.names(ref):
        x = KT.fixture_tensor(ref, name)
        r = _run(fq, x, int(ref["bits/" + name]), task="quantize")
        KT.check_tier_ii(ref, name, x, r.init_ids.cpu().numpy(), float(r.inertia))


def test_resnet18_end_to_end(fq, tmp_path):
    from cnn_quantization_b200 import kmeans_quantization as KQ
    from cnn_quantization_b200 import manager as M
    model = KQ.build_model("resnet18", device="cuda")
    orig = {n: p.detach().clone() for n, p in model.named_parameters()}
    KQ.quantize_model_parameters(model, 4)
    for n, p in model.named_parameters():
        if KQ.is_ignored(n, p):
            assert torch.equal(p, orig[n])
        else:
            assert torch.unique(p).numel() <= 16, n
    p1, p2 = KQ.process_model("resnet18", 4, str(tmp_path), task="quantize")
    assert os.path.basename(p1) == "resnet18_kmeans4bit.pt" and os.path.basename(p2) == "resnet18_kmeans4bit_bcorr.pt"
    mb = torch.load(p2, weights_only=False)
    for n, p in mb.named_parameters():
        if not KQ.is_ignored(n, p):
            w = orig[n].double().view(p.shape[0], -1)
            assert torch.allclose(p.double().view(p.shape[0], -1).mean(1), w.mean(1), rtol=0, atol=1e-6), n
    # evaluation through the manager, weights through DummyQuantizer (qweight='f32')
    args = M.make_args(arch="resnet18", qtype="int8", qweight="f32")
    qm = M.QuantizationManagerInference(args, M.get_params(args))
    qm.enable()
    mq = torch.load(p1, weights_only=False).cuda().eval()
    M.set_node_names(mq)
    M.resnet_mark_before_relu(mq)
    qm.quantize_model(mq)
    qm.attach(mq)
    with torch.no_grad():
        y = mq(torch.randn(2, 3, 64, 64, device="cuda"))
    torch.cuda.synchronize()
    assert y.shape == (2, 1000) and bool(torch.isfinite(y).all())
