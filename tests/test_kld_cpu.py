"""KL-divergence calibration (`-kld`) without a GPU: the numpy restatement (tests/golden/kld_oracle.py) against the
reference's own histograms and divergence curves (tests/golden/ref_kld.npz), the use-mode dispatch with recorders in
place of the launch, the C ABI's argument checks, and the statistics folder the manager picks."""
import ctypes
import os

import numpy as np
import pytest
import torch

import kld_oracle as KO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FP32_EPS = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def ref():
    d = np.load(os.path.join(GOLD, "ref_kld.npz"))
    return {k: d[k] for k in d.files}


def _rows(ref):
    for r in range(len(ref["seed"])):
        yield r, KO.make_row(str(ref["kind"][r]), tuple(int(v) for v in ref["shape"][r]), int(ref["seed"][r]))


def test_oracle_histograms_equal_the_reference(ref):
    for r, x in _rows(ref):
        th, e, h = KO.histogram(x)
        assert np.array_equal(h, ref["hist"][r].astype(np.int64)), ref["kind"][r]
        assert h.sum() == x.size


def test_oracle_threshold_meets_the_divergence_criterion(ref):
    """ref_div[our idx] <= min(ref_div) * (1 + 1e-5) + FP32_EPS; rows whose curve holds NaN choose the reference's index
    and threshold exactly (np.argmin takes the first NaN).

    The absolute term: the reference evaluates sum(P * log(P / Q)) in float32 with sum(P) = 1, so every point of its curve
    carries an absolute error of the order of float32's epsilon from the log ratios alone.  On a nearly degenerate row
    (one non-zero element among 50k zeros) neighbouring candidates differ by less than that, and the reference's pick
    among them is rounding noise."""
    moved = 0
    for r, x in _rows(ref):
        _, e, h = KO.histogram(x)
        th, div, idx = KO.search(h, e)
        curve = ref["div"][r]
        if np.isnan(curve).any():
            assert idx == ref["idx"][r] and th == ref["th"][r], ref["kind"][r]
            continue
        assert curve[idx] <= curve.min() * (1 + 1e-5) + FP32_EPS, (ref["kind"][r], idx, int(ref["idx"][r]))
        moved += idx != ref["idx"][r]
        if idx == ref["idx"][r]:
            assert th == ref["th"][r]
    print("rows with another index than the reference:", moved)


def test_oracle_nan_rows():
    x = np.random.RandomState(0).standard_normal((3, 50)).astype(np.float32)
    x[1, 7] = np.nan
    x[2, 3] = np.inf
    th, div, idx = KO.kld_threshold(x)
    assert np.isfinite(th[0]) and np.isnan(th[1:]).all() and list(idx[1:]) == [-1, -1]


# ---- use-mode dispatch --------------------------------------------------------------------------------------------------
BASE = dict(clipping="no", stats_kind="mean", kld=True, pcq_weights=False, pcq_act=False, bit_alloc_act=False,
            bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
            bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
            logger=None, mtd_quant=False)
STATS = {"min": -1.25, "max": 3.5, "mean": 0.375, "kld_th": 1.7, "b": 0.5, "std": 0.7}


class FakeStats(object):
    def __init__(self, stats):
        self.stats = stats
        self.asked = []

    def get_tensor_stat(self, id, stat, kind):
        self.asked.append((id, stat, kind))
        return np.float64(self.stats[stat])


@pytest.fixture
def recorder(monkeypatch):
    from cnn_quantization_b200 import ops
    calls = []

    def f2g(x, range_, offset, num_bits, int_exp, enforce_true_zero, noise=None, out=None):
        calls.append(("float2gemmlowp", range_, offset, num_bits, enforce_true_zero))
        return torch.zeros_like(x)

    def refuse(name):
        def f(*a, **k):
            calls.append((name,))
            return torch.zeros_like(a[0])
        return f

    monkeypatch.setattr(ops, "float2gemmlowp", f2g)
    for name in ("fused", "quantize1", "quantize1_bca", "kld_threshold"):
        monkeypatch.setattr(ops, name, refuse(name))
    return calls


@pytest.mark.parametrize("half_range", [False, True])
@pytest.mark.parametrize("stats", [STATS, dict(STATS, kld_th=0.5, mean=-0.2), dict(STATS, min=0.25, mean=1.0)])
def test_kld_use_mode_is_one_compiled_leaf_call(recorder, half_range, stats):
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    q = IntQuantizer(4, dict(BASE))
    sm = FakeStats(stats)
    q.sm = lambda: sm
    q.half_range = half_range
    x = torch.randn(2, 8, 4, 4)
    q(x, "conv3_activation", "activation", "conv3_activation")
    q(x, "conv3_activation", "activation", "conv3_activation")   # parameters solved once per layer
    # int_quantizer.py:478-486 + :284-300 + :605-614 in float64 numpy
    if half_range:
        rng, off = np.maximum(np.array(stats["mean"]), 0) + np.float64(stats["kld_th"]), 0
    else:
        rng, off = 2 * np.float64(stats["kld_th"]), np.maximum(np.float64(stats["min"]), stats["mean"] - np.float64(stats["kld_th"]))
    pz = bool((off + rng) > 0 and off < 0)
    assert recorder == [("float2gemmlowp", float(rng), float(off), 4, pz)] * 2
    assert sorted(set(s for _, s, _ in sm.asked)) == ["kld_th", "max", "mean", "min"]
    assert set(k for _, _, k in sm.asked) == {"mean"}
    assert len(sm.asked) == 4


def test_kld_without_statistics_raises(recorder):
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    q = IntQuantizer(4, dict(BASE))
    with pytest.raises(RuntimeError):
        q(torch.randn(2, 8, 4, 4), "conv3_activation", "activation")
    q.sm = lambda: FakeStats(STATS)
    with pytest.raises(RuntimeError):
        q(torch.randn(2, 8, 4, 4), "conv3_activation", "activation")   # no stat_id
    assert recorder == []


def test_kld_leaves_weight_classifier_and_pooling_quantizers_alone(recorder):
    """The manager forces kld off where the reference does (inference_quantization_manager.py:410-473): the same launches
    with and without -kld."""
    from cnn_quantization_b200 import manager
    got = {}
    for kld in (False, True):
        args = manager.make_args(qtype="int4", qweight="int4", kld_threshold=kld)
        qm = manager.QuantizationManagerInference(args, manager.get_params(args))
        assert qm.quantizers["activation"].kld == kld
        del recorder[:]
        for tag, shape in (("weight", (16, 8, 3, 3)), ("weight_classifier", (1000, 64)), ("activation_classifier", (2, 1000)),
                           ("activation_pooling", (2, 8, 4, 4)), ("ignored", (2, 8, 4, 4))):
            q = qm.quantizers[tag]
            assert not q.kld
            q(torch.randn(shape), "x", tag)
        got[kld] = list(recorder)
    assert got[False] == got[True] and len(got[True]) == 5


# ---- C ABI ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


@pytest.mark.parametrize("nb,nq", [(2000, 15), (1, 1), (8003, 15), (0, 15), (2001, 14), (2001, 1), (2001, 2003), (15, 17)])
def test_abi_rejects_bad_bin_counts(lib, nb, nq):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(64)
    rc = lib.fqb200_kld_threshold(buf, 2, 8, nb, nq, buf, buf, buf, buf, 1 << 20, None)
    assert rc == _lib.ERR_INVALID
    assert b"bins" in lib.fqb200_last_error()


def test_abi_workspace_and_sizes(lib):
    from cnn_quantization_b200 import _lib
    assert lib.fqb200_kld_workspace_bytes(512, 2001) >= 512 * 2001 * 4 + 512 * 4
    assert lib.fqb200_kld_workspace_bytes(512, 2000) == 0 and b"num_bins" in lib.fqb200_last_error()
    assert lib.fqb200_kld_workspace_bytes(0, 2001) == 0
    assert lib.fqb200_kld_workspace_bytes(4, 8001) > 0
    buf = ctypes.create_string_buffer(64)
    assert lib.fqb200_kld_threshold(buf, 0, 8, 2001, 15, buf, buf, buf, buf, 1 << 20, None) == _lib.ERR_INVALID
    assert lib.fqb200_kld_threshold(buf, 2, -1, 2001, 15, buf, buf, buf, buf, 1 << 20, None) == _lib.ERR_INVALID
    assert lib.fqb200_kld_threshold(None, 2, 8, 2001, 15, buf, buf, buf, buf, 1 << 20, None) == _lib.ERR_INVALID
    assert lib.fqb200_kld_threshold(buf, 2, 8, 2001, 15, buf, buf, buf, None, 0, None) == _lib.ERR_WORKSPACE


# ---- statistics folder ------------------------------------------------------------------------------------------------------
def test_manager_uses_the_kld_statistics_folder(tmp_path):
    from cnn_quantization_b200 import manager
    args = manager.make_args(qtype="int4", qweight="int8", kld_threshold=True, stats_mode="collect", stats_base_dir=str(tmp_path))
    qm = manager.QuantizationManagerInference(args, manager.get_params(args))
    assert qm.stats_manager.name == "resnet18_kld_int4"
    assert qm.stats_manager.folder == os.path.join(str(tmp_path), "statistics", "resnet18_kld_int4")
    assert qm.stats_manager.stats_names[-7:] == ["mse_lowp", "mse_gaus", "mse_laplace", "cos_lowp", "cos_gaus", "cos_laplace", "kld_th"]
    args = manager.make_args(qtype="int4", qweight="int8", kld_threshold=True, stats_mode="use",
                             stats_base_dir=os.path.join(GOLD, "ref_stats_kld"))
    qm = manager.QuantizationManagerInference(args, manager.get_params(args))
    assert qm._sm_tensor.name == "resnet18_kld_int4"
    assert not np.isnan(qm._sm_tensor.get_tensor_stat("conv1_activation", "kld_th", "mean"))
    # without -kld the folder is the architecture's, and the per-channel manager never gets the column
    args = manager.make_args(qtype="int4", stats_mode="collect", stats_base_dir=str(tmp_path), per_channel_quant_act=True,
                             kld_threshold=True)
    qm = manager.QuantizationManagerInference(args, manager.get_params(args))
    assert "kld_th" not in qm.stats_manager.stats_names
    args = manager.make_args(qtype="int4", stats_mode="collect", stats_base_dir=str(tmp_path))
    assert manager.QuantizationManagerInference(args, manager.get_params(args)).stats_manager.name == "resnet18"
