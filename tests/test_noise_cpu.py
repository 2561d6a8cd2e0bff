"""Quantization-noise measurement (`-ms` with measure_stats_kind="noise") without a GPU: the float64 CPU form against the
reference's own save_measure (tests/golden/make_noise_golden.py), the manager on the seeded ResNet-18 against the
reference manager's files, the manager's rules and the C ABI's argument checks."""
import ctypes
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import fq_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_noise")
W4A4 = dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
            bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)
CONFIGS = {
    "w4a4": W4A4,
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
}
COLUMNS = ["eps_norm", "eps_mse", "eps_cos_sim", "eps_ang_dist", "eps_mean", "eps_var", "w_mean", "w_var", "w_norm",
           "w_size", "x_mean", "x_var", "x_norm", "x_size", "y_mean", "y_var", "y_norm", "y_size", "c_out"]
C = {c: i for i, c in enumerate(COLUMNS)}
# the switches the noise kind turns off: the four every -ms kind turns off, and in-place activations
OFF = ("inplace_activations", "fuse_residual_into_quant", "defer_shortcut", "fuse_pool_into_quant", "fuse_inception_concat")
ON = ("fuse_conv_bias", "skip_redundant_relu", "fuse_residual_relu", "fast_maxpool")


def batches():
    rs = np.random.RandomState(2026)   # make_noise_golden.py's batches: 2 x 4 images, 64x64
    return [torch.from_numpy(rs.standard_normal((4, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


# the angular distance the reference's fp32 cosine makes of a pair at most 16 fp32 rounding steps under 1
ANG_ULPS = float(np.arccos(1.0 - 16 * 2.0 ** -24) / np.pi)


def assert_close_to_reference(got, ref, what):
    """fp32-level agreement with the reference's fp32 arithmetic:
    - sizes and c_out exact, NaN where the reference has NaN;
    - 1e-5 relative on variances and the cosine;
    - a mean within 1e-5 of its tensor's RMS (the reference's fp32 mean is a sum of values of that size, and means of
      signed data sit near 0);
    - norms and the MSE within 1e-5 relative plus n 2^-24 / 64 (times 2 for the MSE, a squared norm), the worst case of
      an fp32 sum of n terms kept in 64 partial sums: the reference's fp32 torch.norm loses accuracy with the element
      count n (3.4e-4 relative measured on a 2.4 M-element weight, 9e-6 on a 65536-element sample);
    - the angular distance within 1e-4 plus ANG_ULPS: arccos amplifies the reference's fp32 cosine near 1, where a pair
      of identical tensors comes out a few fp32 steps under 1 (3.5e-4 measured)."""
    assert got.shape == ref.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(ref)), what
    ok = ~np.isnan(ref)
    g, r = np.where(ok, got, 0.0), np.where(ok, ref, 0.0)
    for name in ("w_size", "x_size", "y_size", "c_out"):
        assert np.array_equal(g[:, C[name]], r[:, C[name]]), (what, name)
    assert np.all(np.abs(g[:, C["eps_ang_dist"]] - r[:, C["eps_ang_dist"]]) <= 1e-4 + ANG_ULPS), what
    size = {"eps": g[:, C["y_size"]], "w": g[:, C["w_size"]], "x": g[:, C["x_size"]], "y": g[:, C["y_size"]]}
    rms = {k: g[:, C[k + "_norm"]] / np.sqrt(size[k]) for k in size}
    for name in COLUMNS:
        if name in ("w_size", "x_size", "y_size", "c_out", "eps_ang_dist"):
            continue
        t, kind = name.split("_")[0], name.split("_")[1]
        rtol = 1e-5 + {"norm": 1, "mse": 2}.get(kind, 0) * size[t] * 2.0 ** -24 / 64
        tol = 1e-5 * rms[t] if kind == "mean" else rtol * np.abs(r[:, C[name]])
        err = np.abs(g[:, C[name]] - r[:, C[name]])
        assert np.all(err <= tol), (what, name, float(np.max(err - tol)))


# ---- the CPU form against the reference's save_measure --------------------------------------------------------------------
def synthetic():
    z = np.load(os.path.join(GOLD, "synthetic.npz"))
    assert list(z["columns"]) == COLUMNS
    names = sorted({k.rsplit("_", 1)[0] for k in z.files if k.endswith("_ref")})
    return {n: tuple(torch.from_numpy(z[n + s]) for s in ("_y", "_yq", "_x", "_w")) + (z[n + "_ref"],) for n in names}


def measure(tmp_path, y, yq, x, w, id="t"):
    from cnn_quantization_b200.statistics import NoiseStatistics
    ms = NoiseStatistics("net", base_dir=str(tmp_path))
    ms.save_measure(y, yq, x, w, id)
    ms.__exit__()
    df = pd.read_csv(os.path.join(str(tmp_path), "noise", "net", id + ".csv"), float_precision="round_trip")
    assert list(df.columns) == COLUMNS
    return df.to_numpy(dtype=np.float64)


@pytest.mark.parametrize("case", ["conv4d", "linear2d", "identical", "large_mean"])
def test_cpu_form_matches_the_reference_save_measure(tmp_path, case):
    y, yq, x, w, ref = synthetic()[case]
    got = measure(tmp_path, y, yq, x, w)
    assert np.array_equal(got, got.astype(np.float32).astype(np.float64), equal_nan=True)   # float32 values
    assert_close_to_reference(got, ref, case)


def test_edge_rules_are_exact(tmp_path):
    y, yq, x, w, ref = synthetic()["conv4d"]
    got = measure(tmp_path, y, yq, x, w)
    assert not y[1].any() and np.isnan(got[1, C["eps_cos_sim"]]) and got[1, C["eps_ang_dist"]] == 0.0   # zero sample
    assert np.isnan(ref[1, C["eps_cos_sim"]]) and ref[1, C["eps_ang_dist"]] == 0.0
    y, yq, x, w, ref = synthetic()["identical"]
    got = measure(tmp_path, y, yq, x, w)
    eps = [C[c] for c in COLUMNS if c.startswith("eps_") and c not in ("eps_cos_sim", "eps_ang_dist")]
    assert not got[:, eps].any() and np.all(got[:, C["eps_cos_sim"]] == 1.0) and not got[:, C["eps_ang_dist"]].any()


def test_cpu_form_sums_and_bias_conventions():
    from cnn_quantization_b200.statistics import sample_noise_cpu
    g = torch.Generator().manual_seed(3)
    y = torch.randn(3, 4, 7, 7, generator=g)
    q = torch.round(y * 2) / 2
    b = torch.randn(4, generator=g)
    yb = y + b.view(1, -1, 1, 1)
    s = sample_noise_cpu(y, q, b, 49)
    yd, qd = yb.reshape(3, -1).double(), q.reshape(3, -1).double()
    want = torch.stack([yd.sum(1), (yd ** 2).sum(1), qd.sum(1), (qd ** 2).sum(1), (yd * qd).sum(1), (yd - qd).sum(1),
                        ((yd - qd) ** 2).sum(1)], 1)
    assert torch.allclose(s, want, rtol=1e-12, atol=1e-9)
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    assert torch.allclose(sample_noise_cpu(cl(y), cl(q), b, -4), want, rtol=1e-12, atol=1e-9)
    yr = y.reshape(3, -1).double()
    assert torch.allclose(sample_noise_cpu(y), torch.stack([yr.sum(1), (yr ** 2).sum(1)], 1))


def test_bn_without_gamma_gives_nan_weight_columns(tmp_path):
    y = torch.randn(2, 3, 4, 4)
    got = measure(tmp_path, y, y, y, None)
    assert np.isnan(got[:, [C["w_mean"], C["w_var"], C["w_norm"], C["w_size"]]]).all()
    assert np.all(got[:, C["c_out"]] == 3) and np.isfinite(got[:, C["x_mean"]]).all()


def test_calls_append_rows_and_the_weight_is_measured_once(tmp_path, monkeypatch):
    from cnn_quantization_b200 import statistics
    from cnn_quantization_b200.statistics import NoiseStatistics
    calls = []
    orig = statistics.sample_noise_cpu
    monkeypatch.setattr(statistics, "sample_noise_cpu", lambda t, *a: (calls.append(tuple(t.shape)), orig(t, *a))[1])
    folder = tmp_path / "noise" / "net"
    folder.mkdir(parents=True)
    (folder / "stale.csv").write_text("x")   # the folder is replaced
    ms = NoiseStatistics("net", base_dir=str(tmp_path))
    w = torch.randn(5, 3)
    ys = [torch.randn(n, 5) for n in (2, 3)]
    for y in ys:
        ms.save_measure(y, y * 0.5, torch.randn(y.shape[0], 3), w, "linear0_activation")
    assert calls.count((1, 15)) == 1   # the weight, as one row, on the first call only
    ms.__exit__()
    assert sorted(os.listdir(str(folder))) == ["linear0_activation.csv"]
    got = pd.read_csv(str(folder / "linear0_activation.csv"), float_precision="round_trip").to_numpy()
    assert got.shape == (5, 19) and np.all(got[:, C["w_size"]] == 15) and np.all(got[:, C["c_out"]] == 5)
    want_norm = np.concatenate([(0.5 * y).norm(dim=1).numpy() for y in ys])
    assert np.allclose(got[:, C["eps_norm"]], want_norm, rtol=1e-6)


def test_nothing_measured_writes_nothing(tmp_path):
    from cnn_quantization_b200.statistics import NoiseStatistics
    NoiseStatistics("net", base_dir=str(tmp_path)).__exit__()
    assert not os.path.exists(os.path.join(str(tmp_path), "noise"))


# ---- the manager on CPU ---------------------------------------------------------------------------------------------------
def fixture(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    assert list(z["columns"]) == COLUMNS
    ids = [str(i) for i in z["ids"]]
    return ids, {k: z["id%03d" % i] for i, k in enumerate(ids)}


def run_resnet18(name, base_dir, capture=None):
    """The seeded ResNet-18 of the fixtures through this package's manager with the noise kind and the CPU oracle's
    quantizers.  ``capture``: a list filled with (id, y, q, x, w) as each call site's measurement got them."""
    from cnn_quantization_b200 import pipeline, statistics
    cfg = dict(arch="resnet18", stats_folder="resnet18", stats_base_dir=base_dir, measure_stats=True,
               measure_stats_kind="noise", **CONFIGS[name])
    model, qm = pipeline.build_quantized_model(cfg, "cpu", quantizer_factory=O.oracle_int_quantizer)
    assert isinstance(qm.measure_stats, statistics.NoiseStatistics)
    if capture is not None:
        orig = statistics.NoiseStatistics.save_measure

        def spy(y, q, x, w, id, bias=None, bias_period=0):
            capture.append((id, y.clone(), q.clone(), x.clone(), w.clone()))
            return orig(qm.measure_stats, y, q, x, w, id, bias, bias_period)

        qm.measure_stats.save_measure = spy
    with torch.no_grad():
        for x in batches():
            model(x)
    qm.__exit__()
    folder = os.path.join(base_dir, "noise", "resnet18")
    return {f[:-4]: pd.read_csv(os.path.join(folder, f), float_precision="round_trip") for f in os.listdir(folder)}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_manager_matches_the_reference_fixture(tmp_path, name):
    torch.set_num_threads(8)   # the generator's: the quantized configs' fp32 convolutions then round alike
    from cnn_quantization_b200.statistics import NoiseStatistics, noise_columns, sample_noise_cpu
    captured = []
    ours = run_resnet18(name, str(tmp_path), capture=captured)
    ids, ref = fixture(name)
    assert sorted(ours) == sorted(ids) and len(ids) == 21
    assert [c[0] for c in captured[:21]] == ids   # call order
    for k in ids:
        assert list(ours[k].columns) == COLUMNS
        got = ours[k].to_numpy(dtype=np.float64)
        assert got.shape == ref[k].shape == (8, 19)
        assert_close_to_reference(got, ref[k], (name, k))
    # the values are the CPU form of exactly the tensors the call sites handed over
    for id, y, q, x, w in captured[:3]:
        n = y.shape[0]
        want = noise_columns(sample_noise_cpu(y, q).numpy(), sample_noise_cpu(x).numpy(),
                             np.tile(sample_noise_cpu(w.reshape(1, -1)).numpy(), (n, 1)), y[0].numel(), x[0].numel(),
                             w.numel(), w.shape[0])
        assert np.array_equal(ours[id].to_numpy(dtype=np.float64)[:n], want), id
    if name == "q_off_int8":
        assert all(torch.equal(y, q) for _, y, q, _, _ in captured)
        assert all(not ours[k][[c for c in COLUMNS[:6] if c not in ("eps_cos_sim",)]].to_numpy().any() for k in ids)
    else:
        assert any(not torch.equal(y, q) for _, y, q, _, _ in captured)


def test_manager_rules(tmp_path):
    from cnn_quantization_b200 import manager as M
    from cnn_quantization_b200.statistics import NoiseStatistics
    mk = lambda **k: M.QuantizationManagerInference(M.make_args(qtype="int4", stats_base_dir=str(tmp_path), **k),
                                                    M.get_params(M.make_args(qtype="int4")))
    dist, noise = mk(measure_stats=True), mk(measure_stats=True, measure_stats_kind="noise")
    assert type(noise.measure_stats) is NoiseStatistics
    assert noise.measure_stats.folder == os.path.join(str(tmp_path), "noise", "resnet18")
    assert mk(measure_stats_kind="noise").measure_stats is None   # the kind alone measures nothing
    plain = mk()
    assert all(getattr(plain, f) for f in OFF + ON)
    assert not any(getattr(noise, f) for f in OFF) and all(getattr(noise, f) for f in ON)
    assert dist.inplace_activations and not any(getattr(dist, f) for f in OFF[1:])
    assert not any(q.inplace for q in noise.quantizers.values() if hasattr(q, "inplace"))
    with pytest.raises(ValueError, match="collect"):
        mk(measure_stats=True, measure_stats_kind="noise", stats_mode="collect")
    with pytest.raises(ValueError, match="measure_stats_kind"):
        mk(measure_stats=True, measure_stats_kind="noisy")


def test_noise_kind_refuses_several_ranks(monkeypatch, tmp_path):
    import torch.distributed as dist
    from cnn_quantization_b200 import manager as M
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    args = M.make_args(qtype="int8", measure_stats=True, measure_stats_kind="noise", stats_base_dir=str(tmp_path))
    with pytest.raises(NotImplementedError):
        M.QuantizationManagerInference(args, M.get_params(args))


# ---- C ABI ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_abi_workspace_bytes(lib):
    f = lib.fqb200_sample_noise_workspace_bytes
    assert f(512, 16384) == 0 and f(7, 49) == 0 and f(0, 100) == 0   # one chunk per row: no partials
    assert f(512, 802816) == 512 * 49 * 7 * 8                        # 64 x 112 x 112: 49 chunks of 16384
    assert f(3, 16385) == 3 * 2 * 7 * 8
    assert f(-1, 100) == 0 and b"rows" in lib.fqb200_last_error()
    assert f(4, 0) == 0 and b"row_len" in lib.fqb200_last_error()


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 16)
    ws = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    need = lib.fqb200_sample_noise_workspace_bytes(2, 20000)
    assert need == 2 * 2 * 7 * 8
    f = lib.fqb200_sample_noise
    assert f(buf, buf, None, 0, -1, 8, buf, None, 0, 0, None) == _lib.ERR_INVALID
    assert f(buf, buf, None, 0, 2, 0, buf, None, 0, 0, None) == _lib.ERR_INVALID
    assert f(None, buf, None, 0, 2, 8, buf, None, 0, 0, None) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error()
    assert f(buf, buf, None, 0, 2, 8, None, None, 0, 0, None) == _lib.ERR_INVALID
    assert f(buf, buf, None, 0, 2, 8, buf, None, 0, -1, None) == _lib.ERR_INVALID
    assert f(buf, buf, buf, 0, 2, 8, buf, None, 0, 0, None) == _lib.ERR_INVALID and b"bias_period" in lib.fqb200_last_error()
    assert f(buf, buf, buf, 3, 2, 8, buf, None, 0, 0, None) == _lib.ERR_INVALID
    assert f(buf, buf, buf, -3, 2, 8, buf, None, 0, 0, None) == _lib.ERR_INVALID
    assert f(buf, buf, buf, 1 << 32, 2, 1 << 33, buf, None, 0, 0, None) == _lib.ERR_UNSUPPORTED
    assert f(buf, buf, None, 0, 2, 20000, buf, None, 0, 0, None) == _lib.ERR_WORKSPACE
    assert f(buf, buf, None, 0, 2, 20000, buf, ws, need - 1, 0, None) == _lib.ERR_WORKSPACE
    assert f(buf, buf, None, 0, 2, 20000, buf, ws + 8, need, 0, None) == _lib.ERR_WORKSPACE
    assert b"workspace" in lib.fqb200_last_error()
    assert f(buf, None, None, 0, 0, 20000, buf, ws, need, 0, None) == _lib.OK   # no rows: nothing is launched
    assert f(buf, buf, buf, 4, 0, 8, buf, None, 0, 7, None) == _lib.OK


def test_ops_refuses_cpu_tensors_and_bad_bias():
    from cnn_quantization_b200 import _lib, ops
    with pytest.raises(_lib.FqError):
        ops.sample_noise(torch.zeros(2, 3))
