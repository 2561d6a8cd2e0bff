"""Activation norm measurement (`-ms`) without a GPU: the C ABI's argument checks, which call sites the manager measures
(against the reference's own distance.csv files, tests/golden/make_distance_golden.py), which tensor it measures, the
three fusions it switches off, and the CSV layout."""
import ctypes
import os

import numpy as np
import pandas as pd
import pytest
import torch
import torch.nn as nn

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_distance")
CONFIGS = {
    "w4a4": dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
                 bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True),
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
    "collect": dict(stats_mode="collect", qtype="int4", qweight="int4"),
}
FUSIONS = ("fuse_residual_into_quant", "defer_shortcut", "fuse_pool_into_quant")
KEPT = ("fuse_conv_bias", "skip_redundant_relu", "fuse_residual_relu", "fast_maxpool", "inplace_activations")


def batches():
    rs = np.random.RandomState(2024)
    return [torch.from_numpy(rs.standard_normal((2, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def fixture(name):
    return pd.read_csv(os.path.join(GOLD, name, "distance.csv"))


# ---- C ABI ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_abi_workspace_bytes(lib):
    assert lib.fqb200_sample_sumsq_workspace_bytes(512, 802816) == 512 * 49 * 8   # 16384-element chunks
    assert lib.fqb200_sample_sumsq_workspace_bytes(512, 16384) == 0               # one chunk per row: no partials
    assert lib.fqb200_sample_sumsq_workspace_bytes(0, 100) == 0
    assert lib.fqb200_sample_sumsq_workspace_bytes(-1, 100) == 0 and b"rows" in lib.fqb200_last_error()
    assert lib.fqb200_sample_sumsq_workspace_bytes(4, 0) == 0 and b"row_len" in lib.fqb200_last_error()


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 12)
    assert lib.fqb200_sample_sumsq(buf, -1, 8, buf, None, 0, None) == _lib.ERR_INVALID
    assert lib.fqb200_sample_sumsq(buf, 2, 0, buf, None, 0, None) == _lib.ERR_INVALID
    assert lib.fqb200_sample_sumsq(buf, 2, -8, buf, None, 0, None) == _lib.ERR_INVALID
    assert lib.fqb200_sample_sumsq(None, 2, 8, buf, None, 0, None) == _lib.ERR_INVALID
    assert b"null" in lib.fqb200_last_error()
    assert lib.fqb200_sample_sumsq(buf, 2, 8, None, None, 0, None) == _lib.ERR_INVALID
    need = lib.fqb200_sample_sumsq_workspace_bytes(2, 40000)
    assert need == 2 * 3 * 8
    assert lib.fqb200_sample_sumsq(buf, 2, 40000, buf, None, 0, None) == _lib.ERR_WORKSPACE
    assert lib.fqb200_sample_sumsq(buf, 2, 40000, buf, buf, need - 1, None) == _lib.ERR_WORKSPACE
    assert b"workspace" in lib.fqb200_last_error()
    assert lib.fqb200_sample_sumsq(buf, 0, 8, buf, None, 0, None) == _lib.OK   # no rows: nothing is launched


# ---- the manager on CPU: recorders in place of the quantization launches -------------------------------------------------
@pytest.fixture
def fake_launches(monkeypatch):
    """ops entry points that return the input unchanged (the native quantizer's dispatch runs; no GPU needed)."""
    from cnn_quantization_b200 import _lib as L, ops

    def fused(x, layout, *, stats_only=False, want_stats=False, out=None, **kw):
        stats = torch.zeros((int(layout[1]), L.STATS_STRIDE))
        if stats_only:
            return stats
        res = x.clone() if out is None else out
        return (res, stats) if want_stats else res

    def same(x, *a, out=None, **k):
        return x.clone() if out is None else out

    monkeypatch.setattr(ops, "fused", fused)
    for name in ("quantize1", "quantize1_bca", "float2gemmlowp"):
        monkeypatch.setattr(ops, name, same)

    def no_gpu(x):
        raise AssertionError("CPU tensors are measured with torch, not ops.sample_sumsq")

    monkeypatch.setattr(ops, "sample_sumsq", no_gpu)


def run_resnet18(flags, base_dir, capture=None):
    """The seeded ResNet-18 of the fixtures, 2 batches of 2 images, through this package's manager; returns the manager
    after __exit__.  ``capture``: (measured, handed_on) lists filled with the tensors save_measure got and the tensors
    the hooked modules handed on."""
    from cnn_quantization_b200 import pipeline, statistics
    cfg = dict(arch="resnet18", stats_folder="resnet18", stats_base_dir=base_dir, measure_stats=True, **flags)
    model, qm = pipeline.build_quantized_model(cfg, "cpu")
    handles = []
    if capture is not None:
        measured, handed_on = capture
        orig = statistics.MeasureStatistics.save_measure
        qm.measure_stats.save_measure = lambda t, id: (measured.append((id, t)), orig(qm.measure_stats, t, id))
        for m in model.modules():
            if type(m) in (nn.Conv2d, nn.Linear):   # registered after the manager's hook: sees what the call site hands on
                handles.append(m.register_forward_hook(lambda m, i, o: handed_on.append(o)))
    with torch.no_grad():
        for x in batches():
            model(x)
    for h in handles:
        h.remove()
    qm.__exit__()
    return qm


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_manager_measures_the_reference_columns(fake_launches, tmp_path, name):
    """Every conv / linear call site in first-call order (torchvision's order inside a block: the shortcut convolution
    last), one row per sample; no poolings, no absorbed BNs, no weights."""
    run_resnet18(CONFIGS[name], str(tmp_path))
    ours = pd.read_csv(os.path.join(str(tmp_path), "distance", "resnet18", "distance.csv"))
    ref = fixture(name)
    assert list(ours.columns) == list(ref.columns)
    assert len(ours) == len(ref) == 4
    assert not any(c.startswith(("maxpool", "avgpool", "bn")) or "weight" in c for c in ours.columns)


@pytest.mark.parametrize("name", ["w4a4", "q_off_int8", "collect"])
def test_the_measured_tensor_is_the_one_the_call_site_hands_on(fake_launches, tmp_path, name):
    measured, handed_on = [], []
    run_resnet18(CONFIGS[name], str(tmp_path), capture=(measured, handed_on))
    assert len(measured) == len(handed_on) == 2 * 21
    assert all(t is o for (_, t), o in zip(measured, handed_on))


def test_bn_sites_are_measured_unless_absorbed(fake_launches, tmp_path):
    from cnn_quantization_b200 import manager as M
    for fold in (False, True):
        args = M.make_args(arch="toy", qtype="int8", qweight="int8", measure_stats=True, stats_base_dir=str(tmp_path))
        qm = M.QuantizationManagerInference(args, M.get_params(args))
        qm.enable()
        try:
            torch.manual_seed(0)
            model = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.MaxPool2d(2), nn.AvgPool2d(2),
                                  nn.Flatten(), nn.Linear(8 * 3 * 3, 10))
        finally:
            qm.stop_stamping()
        if fold:
            M.search_absorbe_bn(model)
            qm.bn_folding = True
        model.eval()
        qm.attach(model)
        with torch.no_grad():
            model(torch.randn(3, 3, 14, 14))
        assert list(qm.measure_stats.stats) == (["conv0_activation", "linear0_activation"] if fold else
                                                ["conv0_activation", "bn0_activation", "linear0_activation"])
        assert all(v[0].shape == (3,) and v[0].dtype == torch.float64 for v in qm.measure_stats.stats.values())
        qm.detach()


def test_fusion_flags_are_off_only_with_measure_stats(tmp_path):
    from cnn_quantization_b200 import manager as M
    for mode in ("no", "collect"):
        plain = M.QuantizationManagerInference(M.make_args(qtype="int4", stats_mode=mode, stats_base_dir=str(tmp_path)),
                                               M.get_params(M.make_args(qtype="int4")))
        ms = M.QuantizationManagerInference(M.make_args(qtype="int4", stats_mode=mode, measure_stats=True,
                                                        stats_base_dir=str(tmp_path)),
                                            M.get_params(M.make_args(qtype="int4")))
        assert plain.measure_stats is None and all(getattr(plain, f) for f in FUSIONS)
        assert ms.measure_stats is not None and not any(getattr(ms, f) for f in FUSIONS)
        assert all(getattr(plain, f) == getattr(ms, f) for f in KEPT)
        assert ms.measure_stats.folder == os.path.join(str(tmp_path), "distance", "resnet18")


def test_measure_stats_refuses_several_ranks(monkeypatch, tmp_path):
    import torch.distributed as dist
    from cnn_quantization_b200 import manager as M
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    args = M.make_args(qtype="int8", measure_stats=True, stats_base_dir=str(tmp_path))
    with pytest.raises(NotImplementedError):
        M.QuantizationManagerInference(args, M.get_params(args))
    M.QuantizationManagerInference(M.make_args(qtype="int8"), M.get_params(args))   # without -ms: unchanged


# ---- the file ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_csv_layout_equals_the_reference(tmp_path, name):
    """Values handed in as samples whose sum of squares is the reference's value come out as the reference's file, byte
    for byte: header, float32 values written as float64, one row per sample, no index."""
    from cnn_quantization_b200.statistics import MeasureStatistics
    ref = fixture(name)
    ms = MeasureStatistics("resnet18", base_dir=str(tmp_path))
    for b in range(2):   # two batches of two samples, as the reference's run
        for col in ref.columns:
            v = torch.tensor(ref[col].to_numpy(dtype=np.float64)[2 * b:2 * b + 2])
            ms.save_measure(v.sqrt().view(2, 1, 1, 1), col)
    ms.__exit__()
    with open(os.path.join(str(tmp_path), "distance", "resnet18", "distance.csv")) as f:
        ours = f.read()
    with open(os.path.join(GOLD, name, "distance.csv")) as f:
        theirs = f.read()
    assert ours.splitlines()[0] == theirs.splitlines()[0]
    assert len(ours.splitlines()) == 5
    assert ours == theirs


def test_nothing_measured_writes_nothing(tmp_path):
    from cnn_quantization_b200.statistics import MeasureStatistics
    MeasureStatistics("resnet18", base_dir=str(tmp_path)).__exit__()
    assert not os.path.exists(os.path.join(str(tmp_path), "distance"))


def test_base_dir_resolution(monkeypatch, tmp_path):
    from cnn_quantization_b200.statistics import MeasureStatistics
    monkeypatch.setenv("FQB200_STATS_DIR", str(tmp_path / "env"))
    assert MeasureStatistics("vgg16").folder == os.path.join(str(tmp_path / "env"), "distance", "vgg16")
    assert MeasureStatistics("vgg16", base_dir=str(tmp_path)).folder == os.path.join(str(tmp_path), "distance", "vgg16")
    monkeypatch.delenv("FQB200_STATS_DIR")
    assert MeasureStatistics("vgg16").folder == os.path.join(os.path.expanduser("~"), "mxt-sim", "distance", "vgg16")


def test_rows_out_of_step_raise(tmp_path):
    from cnn_quantization_b200.statistics import MeasureStatistics
    ms = MeasureStatistics("resnet18", base_dir=str(tmp_path))
    ms.save_measure(torch.ones(2, 3), "conv0_activation")
    ms.save_measure(torch.ones(3, 3), "conv1_activation")
    with pytest.raises(ValueError):
        ms.__exit__()
