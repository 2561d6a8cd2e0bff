"""KL-divergence calibration (`-kld`) on the GPU against the reference's own results (tests/golden/ref_kld.npz,
ref_stats_kld/, ref_stats_kld_logits.npz; made by tests/golden/make_kld_golden.py) and the numpy restatement
(tests/golden/kld_oracle.py)."""
import os

import numpy as np
import pytest
import torch

import kld_oracle as KO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FP32_EPS = float(np.finfo(np.float32).eps)   # absolute noise of the reference's float32 curve (test_kld_cpu.py)


@pytest.fixture(scope="module")
def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(scope="module")
def ref():
    d = np.load(os.path.join(GOLD, "ref_kld.npz"))
    return {k: d[k] for k in d.files}


def _batches(ref):
    """The fixture rows grouped by shape: {shape: (row numbers, [N, C, H, W] cuda tensor)}."""
    groups = {}
    for r in range(len(ref["seed"])):
        shape = tuple(int(v) for v in ref["shape"][r])
        groups.setdefault(shape, []).append(r)
    out = {}
    for shape, rs in groups.items():
        x = np.stack([KO.make_row(str(ref["kind"][r]), shape, int(ref["seed"][r])) for r in rs])
        out[shape] = (rs, torch.from_numpy(x).cuda())
    return out


def test_histograms_bit_exact_nchw_and_channels_last(need_gpu, ref):
    from cnn_quantization_b200 import ops
    for shape, (rs, x) in _batches(ref).items():
        for xin in (x, x.contiguous(memory_format=torch.channels_last)):
            th, div, idx, hist = ops.kld_threshold(xin, return_hist=True)
            h = hist.cpu().numpy()
            for k, r in enumerate(rs):
                assert np.array_equal(h[k], ref["hist"][r]), (ref["kind"][r], shape)


def test_threshold_parity_with_the_reference(need_gpu, ref):
    """ref_div[our idx] <= min(ref_div) * (1 + 1e-5) + float32 eps; NaN curves: the reference's index and threshold."""
    from cnn_quantization_b200 import ops
    moved = []
    for shape, (rs, x) in _batches(ref).items():
        for xin in (x, x.contiguous(memory_format=torch.channels_last)):
            th, div, idx = (t.cpu().numpy() for t in ops.kld_threshold(xin))
            for k, r in enumerate(rs):
                curve = ref["div"][r]
                if np.isnan(curve).any():
                    assert idx[k] == ref["idx"][r] and th[k] == ref["th"][r] and np.isnan(div[k]), ref["kind"][r]
                    continue
                assert curve[idx[k]] <= curve.min() * (1 + 1e-5) + FP32_EPS, (ref["kind"][r], shape, idx[k], ref["idx"][r])
                assert abs(div[k] - curve[idx[k]]) <= 1e-4 * curve[idx[k]] + 4 * FP32_EPS
                if idx[k] == ref["idx"][r]:
                    assert th[k] == ref["th"][r]
                else:
                    moved.append((str(ref["kind"][r]), shape, int(idx[k]), int(ref["idx"][r])))
    print("rows (x2 layouts) with another index than the reference: %d %s" % (len(moved), moved))


def test_nan_and_inf_rows_finish_with_nan(need_gpu):
    from cnn_quantization_b200 import ops
    x = torch.randn(4, 3, 8, 8, device="cuda")
    x[1, 0, 2, 2] = float("nan")
    x[2, 2, 0, 1] = -float("inf")
    th, div, idx = (t.cpu() for t in ops.kld_threshold(x))
    assert torch.isfinite(th[[0, 3]]).all() and torch.isnan(th[[1, 2]]).all() and torch.isnan(div[[1, 2]]).all()
    assert idx[1] == -1 and idx[2] == -1 and idx[0] >= 0
    # odd row lengths take the scalar path; 8001 bins (the MXNet default) fit as well
    y = torch.randn(3, 1001, device="cuda")
    for nb, nq in ((2001, 15), (8001, 15), (2001, 255)):
        th, div, idx, hist = ops.kld_threshold(y, nb, nq, return_hist=True)
        for r in range(3):
            _, e, h = KO.histogram(y[r].cpu().numpy(), nb)
            assert np.array_equal(hist[r].cpu().numpy(), h)
            t, d, i = KO.search(h, e, nq)
            assert int(idx[r]) == i and float(th[r]) == float(t)


def _torch_hist(x2d, nb):
    """[rows, nb] histogram with torch.searchsorted against the same float32 edges (rows of the contiguous [rows, L] view)."""
    rows = x2d.shape[0]
    th = x2d.abs().amax(dim=1).cpu().numpy()
    edges = torch.from_numpy(np.stack([KO.legacy_edges(t, nb) for t in th])).cuda()
    out = torch.zeros((rows, nb), dtype=torch.int64, device="cuda")
    for r in range(rows):
        k = torch.searchsorted(edges[r], x2d[r], right=True) - 1   # e_k <= x < e_{k+1}
        k.clamp_(0, nb - 1)                                          # x == th: the last bin is closed
        out[r] = torch.bincount(k, minlength=nb)
    return out


@pytest.mark.parametrize("name,shape", [("resnet50_stem_n512", (512, 64, 112, 112)), ("vgg16_stem_n672", (672, 64, 224, 224))])
def test_baseline_sizes(need_gpu, name, shape):
    """The ResNet-50 stem activation at N = 512 (411 M elements) and the VGG-16 stem at N = 672 (2.16 G elements > 2^31,
    3.2 M-element rows): histograms equal torch's; the search on 8 rows equals the CPU restatement's."""
    from cnn_quantization_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(shape, device="cuda", generator=g)
    x[1].clamp_(min=0)                   # a ReLU'd sample
    x[2].mul_(3).exp_()                  # a long positive tail
    th, div, idx, hist = ops.kld_threshold(x, return_hist=True)
    x2d = x.view(shape[0], -1)
    sample = list(range(8)) + [shape[0] // 2, shape[0] - 1]
    want = _torch_hist(x2d[sample], 2001)
    assert torch.equal(hist[sample].to(torch.int64), want)
    assert int(hist.to(torch.int64).sum(dim=1).min()) == int(hist.to(torch.int64).sum(dim=1).max()) == x2d.shape[1]
    assert torch.equal(th.cpu(), th.cpu()) and not torch.isnan(th).any()
    h = hist[:8].cpu().numpy()
    amax = x2d[:8].abs().amax(dim=1).cpu().numpy()
    for r in range(8):
        t, d, i = KO.search(h[r], KO.legacy_edges(amax[r], 2001))
        assert int(idx[r]) == i and float(th[r]) == float(t), (r, int(idx[r]), i)
        assert abs(float(div[r]) - d) <= 1e-5 * abs(d) + 1e-9
    del x, x2d, hist


def _run(flags, base_dir, record=False):
    from cnn_quantization_b200 import ops, pipeline
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rs = np.random.RandomState(2024)
    xs = [torch.from_numpy(rs.standard_normal((2, 3, 64, 64)).astype(np.float32)) for _ in range(2)]
    cfg = dict(arch="resnet18", stats_folder="resnet18", stats_base_dir=base_dir, **flags)
    model, qm = pipeline.build_quantized_model(cfg, "cuda")
    outs, prof = [], None
    with torch.no_grad():
        for k, x in enumerate(xs):
            if record and k == 1:
                qm.record, qm.calls = True, []
                ops.profile_reset(enable=True)
            outs.append(model(x.cuda()).cpu().numpy())
            if record and k == 1:
                prof = ops.profile_collect()
                ops.profile_reset(enable=False)
                qm.record = False
    qm.__exit__()
    return np.stack(outs), prof, qm


KLD = dict(qtype="int4", qweight="int8", kld_threshold=True)


def test_resnet18_collect_and_use(need_gpu, tmp_path):
    import pandas as pd
    base = str(tmp_path)
    _run(dict(stats_mode="collect", **KLD), base)
    sub = os.path.join("statistics", "resnet18_kld_int4", "resnet18_kld_int4_summary.csv")
    ours = pd.read_csv(os.path.join(base, sub), index_col=0)
    theirs = pd.read_csv(os.path.join(GOLD, "ref_stats_kld", sub), index_col=0)
    assert list(ours.columns) == list(theirs.columns)
    assert list(ours.index) == list(theirs.index)
    assert list(ours["internal_name"]) == list(theirs["internal_name"])
    for stat in ("min", "max", "mean", "std", "b", "mean_abs", "kurtosis", "dim"):
        for kind in ("min", "mean", "max"):
            col = "%s_%s" % (kind, stat)
            a, b = ours[col].to_numpy(dtype=np.float64), theirs[col].to_numpy(dtype=np.float64)
            scale = np.abs(b).max() + 1e-12
            assert np.allclose(a, b, rtol=2e-3, atol=2e-4 * scale), (col, np.abs(a - b).max())
    # kld_th within one bin width of the layer's largest sample range (2 th / 2001 ~ th / 1000)
    width = np.maximum(theirs["max_max"].abs(), theirs["min_min"].abs()).to_numpy(dtype=np.float64) / 1000
    for kind in ("min", "mean", "max"):
        a = ours["%s_kld_th" % kind].to_numpy(dtype=np.float64)
        b = theirs["%s_kld_th" % kind].to_numpy(dtype=np.float64)
        assert (np.abs(a - b) <= width * 1.0001).all(), (kind, list(ours.index[np.abs(a - b) > width]), np.abs(a - b).max())
    # use mode from the reference's statistics: logits, and one apply-only launch per quantized activation
    got, prof, qm = _run(dict(stats_mode="use", **KLD), os.path.join(GOLD, "ref_stats_kld"), record=True)
    want = np.load(os.path.join(GOLD, "ref_stats_kld_logits.npz"))["use_kld_int4"]
    assert got.shape == want.shape
    cos = float((got * want).sum() / (np.linalg.norm(got) * np.linalg.norm(want)))
    assert cos > 0.97, cos
    assert set(prof["modes"]) - {"E"} == {"A"}, prof["modes"].keys()
    assert prof["modes"]["A"]["launches"] == len(qm.calls) > 0
