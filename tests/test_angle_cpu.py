"""Sample-angle measurement (`-ms` with measure_stats_kind="angle") without a GPU: the C ABI's argument checks, the
manager on the seeded ResNet-18 against the reference's own angle.pkl files (tests/golden/make_angle_golden.py), which
tensor it measures, the fusion flags, and the file's edge cases."""
import ctypes
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import fq_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_angle")
W4A4 = dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
            bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)
CONFIGS = {
    "w4a4": W4A4,
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
    "collect": dict(stats_mode="collect", qtype="int4", qweight="int4"),
}
FUSIONS = ("fuse_residual_into_quant", "defer_shortcut", "fuse_pool_into_quant", "fuse_inception_concat")
# Against the reference's angle.pkl.  Where no activation is quantized (q_off_int8, collect) only fp32 round-off of the CPU
# convolutions and the reference's fp32 cosine differ: the largest deviation measured was 4.3e-6 rad, over 1 to 32 host
# threads and the AVX-512, AVX2 and SSE4 kernels of torch.  Where activations are quantized, the CPU's fp32 sums depend on
# the thread count and the instruction set, and a last-ulp difference can move a value across a rounding boundary of the
# quantization grid: one grid step of one element, which then propagates.  Measured: with 1, 3 or 4 threads one 8-bit step
# of one W4A4 logit (3.5e-5 rad); with AVX2 or SSE4 kernels steps in the convolution outputs (0.036 rad W4A4, 0.0034 rad
# W8A8; the GPU run of the same model shows 0.035 and 0.0049).  The bound there is the repo's parity figure for quantized
# runs, each tensor within 10 % of the reference's (test_gpu_pipeline.py): a relative perturbation e of each of two vectors
# moves their angle by at most 2 asin(e) = 0.2 rad.  The values themselves are pinned exactly, on every host, to the
# float64 form applied to the tensors the call sites handed on.
REF_BOUND = {"q_off_int8": 1e-5, "collect": 1e-5, "w4a4": 0.2, "w8a8": 0.2}


def batches():
    rs = np.random.RandomState(2025)   # make_angle_golden.py's batches: 2 x 6 images, 64x64
    return [torch.from_numpy(rs.standard_normal((6, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def fixture(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    ids = [str(i) for i in z["ids"]]
    return ids, {k: z["id%03d" % i] for i, k in enumerate(ids)}, z["target"]


# ---- C ABI ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_abi_workspace_bytes(lib):
    # 512 rows: 8 tiles, 36 tile pairs; 802816 elements = 25088 k-steps of 32, cut into ceil(1024 / 36) = 29 slices
    assert lib.fqb200_sample_angles_workspace_bytes(512, 802816) == 36 * 29 * 64 * 64 * 8
    # a short row: as many slices as 8-step slices fit (49 elements: 2 steps, one slice)
    assert lib.fqb200_sample_angles_workspace_bytes(7, 49) == 64 * 64 * 8
    assert lib.fqb200_sample_angles_workspace_bytes(1, 100352) == 392 * 64 * 64 * 8
    assert lib.fqb200_sample_angles_workspace_bytes(0, 100) == 0
    # the slice count depends on the shape only: at the row limit every pair is one unit
    assert lib.fqb200_sample_angles_workspace_bytes(8192, 802816) == 128 * 129 // 2 * 64 * 64 * 8
    assert lib.fqb200_sample_angles_workspace_bytes(-1, 100) == 0 and b"rows" in lib.fqb200_last_error()
    assert lib.fqb200_sample_angles_workspace_bytes(4, 0) == 0 and b"row_len" in lib.fqb200_last_error()
    assert lib.fqb200_sample_angles_workspace_bytes(8193, 4) == 0 and b"8192" in lib.fqb200_last_error()


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 16)
    need = lib.fqb200_sample_angles_workspace_bytes(2, 8)
    assert need == 64 * 64 * 8
    f = lib.fqb200_sample_angles
    assert f(buf, -1, 8, buf, None, buf, need, 0, None) == _lib.ERR_INVALID
    assert f(buf, 2, 0, buf, None, buf, need, 0, None) == _lib.ERR_INVALID
    assert f(buf, 2, -8, buf, None, buf, need, 0, None) == _lib.ERR_INVALID
    assert f(buf, 2, 8, None, None, buf, need, 0, None) == _lib.ERR_INVALID
    assert b"out_angles and out_gram" in lib.fqb200_last_error()
    assert f(None, 2, 8, buf, None, buf, need, 0, None) == _lib.ERR_INVALID
    assert b"null" in lib.fqb200_last_error()
    assert f(buf, 2, 8, buf, None, buf, need, -1, None) == _lib.ERR_INVALID
    assert f(buf, 2, 8, buf, None, None, 0, 0, None) == _lib.ERR_WORKSPACE
    assert f(buf, 2, 8, buf, buf, buf, need - 1, 0, None) == _lib.ERR_WORKSPACE
    assert b"workspace" in lib.fqb200_last_error()
    assert f(buf, 8193, 8, buf, None, buf, need, 0, None) == _lib.ERR_UNSUPPORTED
    assert f(buf, 0, 8, buf, None, None, 0, 0, None) == _lib.OK   # no rows: nothing is launched


# ---- the CPU form -------------------------------------------------------------------------------------------------------------
def test_cpu_form_special_cases():
    from cnn_quantization_b200.statistics import sample_angles_cpu
    x = torch.randn(6, 3, 5, 5, dtype=torch.float64).float()
    x[1] = x[0]
    x[2] = -x[0]
    x[3] = 0
    x[4, 0, 0, 0] = float("inf")
    a = sample_angles_cpu(x)
    assert a.dtype == torch.float32 and a.shape == (6, 6)
    assert torch.equal(torch.tril(a), torch.zeros(6, 6))
    assert abs(float(a[0, 2]) - float(np.float32(np.pi))) <= float(np.spacing(np.float32(np.pi)))
    assert float(a[0, 1]) < 1e-6
    assert torch.isnan(a[:3, 3]).all() and torch.isnan(a[3, 4:]).all()
    assert torch.isnan(a[:4, 4]).all() and torch.isnan(a[4, 5])
    assert torch.isfinite(a[0, 5]) and torch.isfinite(a[2, 5])


# ---- the manager on CPU -------------------------------------------------------------------------------------------------------
@pytest.fixture
def fake_launches(monkeypatch):
    """ops entry points that return the input unchanged (collect mode's native quantizer dispatch runs; no GPU needed)."""
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

    def no_gpu(x, *a, **k):
        raise AssertionError("CPU tensors are measured with torch, not ops.sample_angles")

    monkeypatch.setattr(ops, "sample_angles", no_gpu)


def run_resnet18(name, base_dir, capture=None, angles=None):
    """The seeded ResNet-18 of the fixtures through this package's manager with the angle kind: the CPU oracle's
    quantizers, or (collect mode, which quantizes no activation) the native dispatch with the launches faked.  Returns the
    pickle.  ``capture``: (measured, handed_on) lists filled with the tensors save_measure got and the tensors the hooked
    modules handed on.  ``angles``: a dict filled with {id: [the CPU form's matrix of what the call site handed on]},
    computed in the hook, before any later in-place write."""
    from cnn_quantization_b200 import pipeline, statistics
    cfg = dict(arch="resnet18", stats_folder="resnet18", stats_base_dir=base_dir, measure_stats=True,
               measure_stats_kind="angle", **CONFIGS[name])
    factory = None if name == "collect" else O.oracle_int_quantizer
    model, qm = pipeline.build_quantized_model(cfg, "cpu", quantizer_factory=factory)
    assert isinstance(qm.measure_stats, statistics.AngleStatistics)
    handles = []
    if capture is not None:
        measured, handed_on = capture
        orig = statistics.AngleStatistics.save_measure
        qm.measure_stats.save_measure = lambda t, id: (measured.append((id, t)), orig(qm.measure_stats, t, id))
        for m in model.modules():
            if type(m) in (nn.Conv2d, nn.Linear):   # registered after the manager's hook: sees what the call site hands on
                handles.append(m.register_forward_hook(lambda m, i, o: handed_on.append(o)))
    if angles is not None:
        def oracle(m, i, o):   # registered after the manager's hook
            prefix = "conv" if isinstance(m, nn.Conv2d) else "linear"
            angles.setdefault("%s%d_activation" % (prefix, m._fq_id), []).append(statistics.sample_angles_cpu(o))

        handles += [m.register_forward_hook(oracle) for m in model.modules() if type(m) in (nn.Conv2d, nn.Linear)]
    with torch.no_grad():
        for x in batches():
            model(x)
    for h in handles:
        h.remove()
    qm.__exit__()
    with open(os.path.join(base_dir, "angle", "resnet18", "angle.pkl"), "rb") as f:
        return pickle.load(f)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_manager_matches_the_reference_fixture(fake_launches, tmp_path, name):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    handed_on = {}
    ours = run_resnet18(name, str(tmp_path), angles=handed_on)
    ids, ref, target = fixture(name)
    assert list(ours) == ids + ["target"]
    assert isinstance(ours["target"], list) and ours["target"] == [] and target.size == 0
    worst = 0.0
    for k in ids:
        got = ours[k].to_numpy()
        assert got.dtype == np.float64 and got.shape == ref[k].shape == (12, 6)
        for b in range(2):
            blk, rblk = got[6 * b:6 * b + 6], ref[k][6 * b:6 * b + 6]
            assert np.array_equal(np.tril(blk), np.zeros((6, 6))) and np.array_equal(np.tril(rblk), np.zeros((6, 6)))
        assert np.array_equal(got, got.astype(np.float32).astype(np.float64))   # float32 values
        assert np.array_equal(got, torch.cat(handed_on[k]).numpy().astype(np.float64)), k
        err = float(np.max(np.abs(got - ref[k])))
        worst = max(worst, err)
        assert err < REF_BOUND[name], (k, err)
    print("%s: largest deviation from the reference %.3g rad" % (name, worst))


@pytest.mark.parametrize("name", ["w4a4", "q_off_int8", "collect"])
def test_the_measured_tensor_is_the_one_the_call_site_hands_on(fake_launches, tmp_path, name):
    measured, handed_on = [], []
    run_resnet18(name, str(tmp_path), capture=(measured, handed_on))
    assert len(measured) == len(handed_on) == 2 * 21
    assert all(t is o for (_, t), o in zip(measured, handed_on))


def test_fusion_flags_are_off_as_with_the_norm_kind(tmp_path):
    from cnn_quantization_b200 import manager as M
    from cnn_quantization_b200.statistics import AngleStatistics, MeasureStatistics
    for mode in ("no", "collect"):
        mk = lambda **k: M.QuantizationManagerInference(M.make_args(qtype="int4", stats_mode=mode, stats_base_dir=str(tmp_path), **k),
                                                        M.get_params(M.make_args(qtype="int4")))
        dist, ang = mk(measure_stats=True), mk(measure_stats=True, measure_stats_kind="angle")
        assert type(dist.measure_stats) is MeasureStatistics and type(ang.measure_stats) is AngleStatistics
        assert all(getattr(dist, f) == getattr(ang, f) for f in FUSIONS) and not any(getattr(ang, f) for f in FUSIONS)
        assert ang.measure_stats.folder == os.path.join(str(tmp_path), "angle", "resnet18")
        assert mk(measure_stats_kind="angle").measure_stats is None   # the kind alone measures nothing


def test_angle_kind_refuses_several_ranks(monkeypatch, tmp_path):
    import torch.distributed as dist
    from cnn_quantization_b200 import manager as M
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    args = M.make_args(qtype="int8", measure_stats=True, measure_stats_kind="angle", stats_base_dir=str(tmp_path))
    with pytest.raises(NotImplementedError):
        M.QuantizationManagerInference(args, M.get_params(args))


def test_unknown_kind_raises(tmp_path):
    from cnn_quantization_b200 import manager as M
    args = M.make_args(qtype="int8", measure_stats=True, measure_stats_kind="cosine", stats_base_dir=str(tmp_path))
    with pytest.raises(ValueError, match="measure_stats_kind"):
        M.QuantizationManagerInference(args, M.get_params(args))


# ---- the file -----------------------------------------------------------------------------------------------------------------
def test_mismatched_sample_count_names_the_id(tmp_path):
    from cnn_quantization_b200.statistics import AngleStatistics
    ms = AngleStatistics("resnet18", base_dir=str(tmp_path))
    ms.save_measure(torch.ones(4, 3), "conv0_activation")
    ms.save_measure(torch.ones(3, 3), "conv1_activation")   # another id may see another N
    with pytest.raises(ValueError, match="conv0_activation"):
        ms.save_measure(torch.ones(5, 3), "conv0_activation")


def test_nothing_measured_writes_nothing(tmp_path):
    from cnn_quantization_b200.statistics import AngleStatistics
    ms = AngleStatistics("resnet18", base_dir=str(tmp_path))
    ms.save_target(torch.tensor([1, 2]))
    ms.__exit__()
    assert not os.path.exists(os.path.join(str(tmp_path), "angle"))


def test_file_layout_and_targets(tmp_path):
    from cnn_quantization_b200.statistics import AngleStatistics
    folder = tmp_path / "angle" / "resnet18"
    folder.mkdir(parents=True)
    (folder / "stale.txt").write_text("x")   # the folder is removed and recreated
    ms = AngleStatistics("resnet18", base_dir=str(tmp_path))
    xs = [torch.randn(3, 2, 4, 4) for _ in range(2)]
    for x in xs:
        ms.save_measure(x, "conv1_activation")
        ms.save_measure(x[:, :1], "conv0_activation")
        ms.save_target(torch.tensor([3, 1, 4]))
    ms.__exit__()
    assert sorted(os.listdir(str(folder))) == ["angle.pkl"]
    with open(str(folder / "angle.pkl"), "rb") as f:
        d = pickle.load(f)
    assert list(d) == ["conv1_activation", "conv0_activation", "target"]
    assert d["conv1_activation"].shape == (6, 3) and list(d["conv1_activation"].columns) == [0, 1, 2]
    assert d["target"].dtype == np.float64 and d["target"].tolist() == [3, 1, 4, 3, 1, 4]
    from cnn_quantization_b200.statistics import sample_angles_cpu
    want = np.vstack([sample_angles_cpu(x).numpy() for x in xs]).astype(np.float64)
    assert np.array_equal(d["conv1_activation"].to_numpy(), want)
